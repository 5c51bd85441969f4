"""The current scan's deskewed cloud and the record index of every point (Pipeline(keep_cloud=True),
currentCloudArray / currentCloudIndices, madtree_gpu_cloud*).  The cloud is the reference's curr_cloud
(odometry/pipeline.cpp:140): after the gate, the correction and the deskew, before MADtree reorders it.  Every check is
bit for bit: against the oracle's Pipeline::deskew, the host restatements of the gate, the correction and the time-stamp
deskew, numpy's iso_apply, and across every ingest path."""
import ctypes as C
import os

import numpy as np
import pytest

from mad_icp_b200 import _capi, records, synth
from util import bits_equal

KITTI_GATE = dict(min_range=0.7, max_range=120.0, inclusive=True, drop_nan=False)
OUSTER_GATE = dict(min_range=1.3, max_range=120.0, inclusive=False, drop_nan=True)
OUSTER = np.dtype({"names": ["x", "y", "z", "intensity", "t", "reflectivity"],
                   "formats": ["<f4", "<f4", "<f4", "<f4", "<u4", "<u2"], "offsets": [0, 4, 8, 16, 20, 40], "itemsize": 48})
T_PREV = synth.pose_xyyaw(0.0, 0.0, 0.0)
T_NOW = synth.pose_xyyaw(0.8, 0.05, 0.03)
NEW_SYMBOLS = ["madicp_set_keep_cloud", "madtree_gpu_num_cloud_points", "madtree_gpu_cloud", "madtree_gpu_cloud_dev",
               "madtree_gpu_release_cloud"]
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_symbols_bound(built):
    L = _capi.lib()
    for name in NEW_SYMBOLS:
        assert name in _capi.SYMBOLS and getattr(L, name).restype is not None
    assert L.madicp_abi_version() > 0


def test_bad_arguments_without_gpu(built):
    L = _capi.lib()
    xyz, idx = np.empty((4, 3)), np.empty(4, np.int64)
    assert L.madicp_set_keep_cloud(None, 1) < 0
    assert L.madtree_gpu_num_cloud_points(None) < 0
    assert L.madtree_gpu_cloud(None, None, _capi.as_d(xyz), idx.ctypes.data_as(C.POINTER(C.c_int64))) < 0
    assert b"null tree" in L.madicp_last_error()
    assert L.madtree_gpu_cloud_dev(None, None, None, None, None) < 0
    assert L.madtree_gpu_release_cloud(None) < 0


# ----------------------------------------------------------------------------------------------------------- helpers
def _pipeline(hz=10.0, deskew=True, keep=True, gpu_build=True):
    from mad_icp_b200.pybind.pypeline import Pipeline
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        return Pipeline(sensor_hz=hz, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                        num_keyframes=4, num_threads=4, realtime=False, keep_cloud=keep)
    finally:
        os.environ.pop("MADICP_GPU_BUILD")


def _sequence(n, layout="kitti"):
    """KITTI float32 N x 4 records or Ouster 48-byte records (NaN rows among them), on a street"""
    scene = synth.StreetScene(seed=7, x_min=-45.0, x_max=60.0 + 0.8 * n)
    out = []
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.3 * np.sin(0.05 * i), 0.02 * np.sin(0.03 * i))
        p = synth.lidar_scan(scene, base, beams=32, azimuths=1024, seed=100 + i, r_min=0.0, r_max=np.inf)
        rs = np.random.RandomState(i)
        p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=p.shape[0] // 20)), np.nan, axis=0)
        if layout == "kitti":
            a = np.zeros((p.shape[0], 4), np.float32)
            a[:, :3] = p
            a[:, 3] = np.linspace(-0.1, 0.0, p.shape[0])
        else:
            a = np.zeros(p.shape[0], OUSTER)
            a["x"], a["y"], a["z"] = p[:, 0], p[:, 1], p[:, 2]
            a["t"] = np.linspace(0, 99_000_000, p.shape[0]).astype(np.uint32)
        out.append(a)
    return out


def _xyz(a):
    return np.column_stack([a["x"], a["y"], a["z"]]) if a.dtype.names else np.asarray(a[:, :3])


def _kept(a, gate, correction=False):
    """the reader's kept points (float64, corrected like KittiReader) and their record indices"""
    mask = records.range_mask(a, **gate).astype(bool)
    pts = records.correct_vertical_angle(a, **gate) if correction else _xyz(a)[mask].astype(np.float64)
    return pts, np.flatnonzero(mask)


def _azimuth_perm(a, gate, hz, T_prev, T_now, correction=False):
    d = records.describe(a, **gate)
    v = records.vcorr(correction)
    perm, chunk, poses = np.empty(d.n, np.int32), np.empty(d.n, np.uint16), np.empty((2048, 12))
    n_poses, kept = C.c_int(0), C.c_int64(0)
    _capi.check(_capi.lib().madicp_debug_deskew_plan(C.byref(d), C.byref(v) if v else None, _capi.as_d(_capi.pose12(T_prev)),
                                                     _capi.as_d(_capi.pose12(T_now)), hz, 0, 4, _capi.as_i(perm),
                                                     chunk.ctypes.data_as(C.POINTER(C.c_uint16)), _capi.as_d(poses),
                                                     C.byref(n_poses), C.byref(kept)), "madicp_debug_deskew_plan")
    return perm[:kept.value].astype(np.int64)


def _iso_apply(T, p):
    """X * p with iso_apply's operand order: ((r0 x + r1 y) + r2 z) + t, no FMA"""
    X = np.asarray(T, np.float64)[:3]
    return ((X[None, :, 0] * p[:, 0:1] + X[None, :, 1] * p[:, 1:2]) + X[None, :, 2] * p[:, 2:3]) + X[None, :, 3]


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=4)


@gpu
def test_keep_off_empty_and_bad_frame(built):
    from mad_icp_b200.pybind.pypeline import MadIcpError
    off = _pipeline(keep=False)
    for call in (lambda: off.currentCloudArray(), lambda: off.currentCloudIndices(), lambda: off.currentCloudArray(device=True)):
        with pytest.raises(MadIcpError, match="keep_cloud"):
            call()
    p = _pipeline()
    with pytest.raises(ValueError):
        p.currentCloudArray(frame="world")
    assert p.currentCloudArray().shape == (0, 3) and p.currentCloudIndices().shape == (0,)
    assert p.currentCloudIndices().dtype == np.int64
    assert tuple(p.currentCloudArray(device=True).shape) == (0, 3)


@gpu
def test_trees_without_a_cloud_and_bad_outputs(reg):
    import torch
    L = _capi.lib()
    pts = _kept(_sequence(1)[0], KITTI_GATE)[0]
    reg.keep_cloud(False)
    t = reg.build_tree(pts)
    assert L.madtree_gpu_num_cloud_points(t._h) == -3  # MADICP_ERR_STATE
    with pytest.raises(_capi.MadIcpError, match="kept no cloud"):
        t.cloud()
    reg.keep_cloud(True)
    try:
        t = reg.build_tree(pts)
        assert L.madtree_gpu_num_cloud_points(t._h) == pts.shape[0]
        xyz, idx = t.cloud()
        assert bits_equal(xyz, pts) and (idx == np.arange(pts.shape[0])).all()
        host = np.empty((pts.shape[0], 3))
        assert L.madtree_gpu_cloud_dev(t._h, None, C.c_void_p(host.ctypes.data), None, None) < 0  # host memory
        assert b"device memory" in L.madicp_last_error()
        buf = torch.empty(pts.shape[0] * 3 + 1, dtype=torch.float64, device="cuda")
        assert L.madtree_gpu_cloud_dev(t._h, None, C.c_void_p(buf.data_ptr() + 4), None, None) < 0  # misaligned
        assert b"aligned" in L.madicp_last_error()
        assert L.madtree_gpu_cloud(t._h, None, None, None) < 0  # no output
        t.release_cloud()
        assert L.madtree_gpu_num_cloud_points(t._h) == -3
    finally:
        reg.keep_cloud(False)


@gpu
def test_every_ingest_path_of_the_engine(reg):
    """Registrar-level: every ingest path keeps the cloud it built from and the record indices, forests included."""
    import torch
    seq = _sequence(4)
    reg.keep_cloud(True)
    try:
        a = seq[0]
        kept, rec = _kept(a, KITTI_GATE)
        dsk = dict(deskew=True, T_prev=T_PREV, T_now=T_NOW, sensor_hz=10.0)
        perm = _azimuth_perm(a, KITTI_GATE, 10.0, T_PREV, T_NOW)

        def same(want, idx, what):  # the tree of the cloud the ingest just left keeps exactly that cloud
            xyz, got = reg.build_tree().cloud()
            assert bits_equal(xyz, want) and (got == idx).all(), what

        for src in (a, torch.from_numpy(a).cuda()):  # host records, device records
            same(reg.ingest_records(src, **KITTI_GATE, want_points=True), rec, "gated")
            same(reg.ingest_records(src, **KITTI_GATE, want_points=True, **dsk), perm, "azimuth")
            same(reg.ingest_records(src, **KITTI_GATE, want_points=True, time_field=3, **dsk), rec, "time")
            for idx_want, kw in ((perm, {}), (rec, dict(time_field=3))):
                plan = reg.plan_records(src, **KITTI_GATE, **kw)
                same(reg.ingest_plan(plan, want_points=True, **dsk), idx_want, ("plan", kw))
                plan = reg.plan_records(src, **KITTI_GATE, **kw)  # consumed without a deskew
                same(reg.ingest_plan(plan, want_points=True), rec, ("plan, no deskew", kw))
        packed = np.ascontiguousarray(kept, np.float32)
        same(reg.ingest(packed, want_points=True), np.arange(kept.shape[0]), "packed")
        same(reg.ingest(packed, want_points=True, **dsk), _azimuth_perm(packed, {}, 10.0, T_PREV, T_NOW), "packed, azimuth")
        # forests: packed clouds (record = row), host records, device records -- each tree its own slice
        outs = [_kept(s, KITTI_GATE) for s in seq]
        for trees, rows in ((reg.build_trees([o[0] for o in outs]), True), (reg.build_trees_records(seq, **KITTI_GATE), False),
                            (reg.build_trees_records([torch.from_numpy(s).cuda() for s in seq], **KITTI_GATE), False)):
            for t, (want, rec_b) in zip(trees, outs):
                xyz, idx = t.cloud()
                assert bits_equal(xyz, want) and (idx == (np.arange(want.shape[0]) if rows else rec_b)).all()
        # posed output and the device form
        t = trees[2]
        T = synth.pose_xyyaw(3.0, -1.0, 0.4, z=0.2)
        xyz, idx = t.cloud(T)
        assert bits_equal(xyz, _iso_apply(T, outs[2][0]))
        dx, di = t.cloud(T, device=True)
        assert bits_equal(dx.cpu().numpy(), xyz) and (di.cpu().numpy() == idx).all()
    finally:
        reg.keep_cloud(False)


def _check_deskewed_sequence(oracle, layout, gate, correction, hz, n=40):
    seq = _sequence(n, layout)
    p = _pipeline(hz)
    ties = 0
    for i, a in enumerate(seq):
        T = p.trajectory()
        p.computeRecords(0.1 * i, a, **gate, apply_correction=correction)
        kept, rec = _kept(a, gate, correction)
        got, idx = p.currentCloudArray(frame="sensor"), p.currentCloudIndices()
        if len(T) < 2:  # the first two scans are not deskewed
            assert bits_equal(got, kept) and (idx == rec).all(), i
            continue
        assert bits_equal(got, oracle.deskew(kept, T[-2], T[-1], hz)), i
        assert (idx == _azimuth_perm(a, gate, hz, T[-2], T[-1], correction)).all(), i
        az = np.arctan2(kept[:, 1], kept[:, 0])
        ties += az.size - np.unique(az).size
    assert ties > 0  # scans with tied azimuths were among them


@gpu
@pytest.mark.parametrize("hz", [10.0, 20.0])
@pytest.mark.parametrize("layout,gate,correction", [("kitti", KITTI_GATE, False), ("kitti", KITTI_GATE, True),
                                                    ("ouster", OUSTER_GATE, False), ("ouster", OUSTER_GATE, True)])
def test_azimuth_deskew_is_the_reference(oracle, layout, gate, correction, hz):
    _check_deskewed_sequence(oracle, layout, gate, correction, hz)


@gpu
@pytest.mark.parametrize("layout,gate", [("kitti", KITTI_GATE), ("ouster", OUSTER_GATE)])
def test_no_deskew_is_the_readers_array(built, layout, gate):
    p = _pipeline(deskew=False)
    for i, a in enumerate(_sequence(6, layout)):
        p.computeRecords(0.1 * i, a, **gate)
        kept, rec = _kept(a, gate)
        assert bits_equal(p.currentCloudArray(frame="sensor"), kept) and (p.currentCloudIndices() == rec).all()
        if layout == "ouster":
            assert np.isnan(_xyz(a)).any(axis=1).sum() > 0 and not np.isin(np.flatnonzero(np.isnan(_xyz(a)).any(axis=1)), rec).any()


@gpu
@pytest.mark.parametrize("layout,gate,field,scale", [("kitti", KITTI_GATE, 3, 1.0), ("ouster", OUSTER_GATE, "t", 1e-9)])
def test_time_deskew_is_the_restatement(built, layout, gate, field, scale):
    hz = 10.0
    p = _pipeline(hz)
    for i, a in enumerate(_sequence(8, layout)):
        T = p.trajectory()
        p.computeRecords(0.1 * i, a, **gate, time_field=field, time_scale=scale)
        kept, rec = _kept(a, gate)
        want = kept
        if len(T) >= 2:
            k = records.time_chunks(a, field, scale, hz, **gate)
            P = records.chunk_poses(T[-2], T[-1], hz)
            R, t = P[k, :, :3], P[k, :, 3]
            want = ((R[:, :, 0] * kept[:, None, 0] + R[:, :, 1] * kept[:, None, 1]) + R[:, :, 2] * kept[:, None, 2]) + t
        assert bits_equal(p.currentCloudArray(frame="sensor"), want) and (p.currentCloudIndices() == rec).all(), i


@gpu
def test_map_frame_and_the_first_scan(built):
    seq = _sequence(6)
    seq[0][np.flatnonzero(records.range_mask(seq[0], **KITTI_GATE))[5], 2] = -0.0
    for gpu_build in (True, False):
        p = _pipeline(deskew=False, gpu_build=gpu_build)
        for i, a in enumerate(seq):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
            sensor, world = p.currentCloudArray(frame="sensor"), p.currentCloudArray()
            if i == 0:  # no pose yet: the sensor bits, -0.0 included
                assert bits_equal(world, sensor) and np.signbit(world[5, 2]) and world[5, 2] == 0.0
            else:
                assert bits_equal(world, _iso_apply(p.currentPose(), sensor)), (gpu_build, i)


def _run(seq, mode, deskew, keep=True, depth=0, shift=0):
    """a whole sequence through one ingest path; returns what the pipeline hands out after every scan"""
    import torch
    p = _pipeline(deskew=deskew, keep=keep, gpu_build=mode != "host")
    gated = [_kept(a, KITTI_GATE)[0] for a in seq]
    out, queued = [], 0
    for i, a in enumerate(seq):
        if mode == "prefetch":
            while queued < min(i + depth, len(seq)):
                assert p.prefetchRecords(seq[queued], **KITTI_GATE, deskew_ahead=deskew)
                queued += 1
        if mode == "prefetch_f32":
            while queued < min(i + depth, len(seq)):
                assert p.prefetch(gated[queued].astype(np.float32), deskew_ahead=deskew)
                queued += 1
        if mode in ("records", "host", "prefetch"):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
        elif mode == "cuda":
            raw = np.frombuffer(a.tobytes(), np.uint8)
            buf = torch.zeros(raw.size + 64, dtype=torch.uint8, device="cuda")
            buf[shift:shift + raw.size] = torch.from_numpy(raw.copy()).cuda()
            p.computeRecords(0.1 * i, buf[shift:shift + raw.size].view(torch.float32).view(-1, 4), **KITTI_GATE)
        elif mode in ("f32", "prefetch_f32"):
            p.compute(0.1 * i, gated[i].astype(np.float32))
        elif mode == "f64":
            p.compute(0.1 * i, gated[i])
        elif mode == "vec":
            from mad_icp_b200.pybind.pypeline import VectorEigen3d
            p.compute(0.1 * i, VectorEigen3d(gated[i]))
        o = dict(pose=p.currentPose().copy(), kf=int(p.keyframeID()), inl=float(p.inliersRatio()))
        if keep:
            o.update(sensor=p.currentCloudArray(frame="sensor"), map=p.currentCloudArray(), idx=p.currentCloudIndices())
            if mode not in ("records", "host", "prefetch", "cuda"):  # the packed arrays' rows -> the records'
                o["idx"] = _kept(a, KITTI_GATE)[1][o["idx"]]
        out.append(o)
    return out


def _same(got, want, what):
    for i, (g, w) in enumerate(zip(got, want)):
        for k in w:
            if k in g:
                assert (bits_equal(g[k], w[k]) if isinstance(w[k], np.ndarray) else g[k] == w[k]), (what, i, k)


@gpu
@pytest.mark.parametrize("deskew", [False, True])
def test_same_bits_on_every_path(built, deskew):
    seq = _sequence(30)
    want = _run(seq, "records", deskew)
    assert sum(1 for i in range(1, len(want)) if want[i]["kf"] != want[i - 1]["kf"]) >= 1
    _same(_run(seq, "records", deskew, keep=False), want, "keep off")  # registration is unchanged
    for mode in ("f32", "f64", "vec", "host"):
        _same(_run(seq, mode, deskew), want, mode)
    for shift in (4, 8, 12):
        _same(_run(seq, "cuda", deskew, shift=shift), want, ("cuda", shift))
    for depth in (1, 5, 32):  # with later scans prefetched, each scan's own cloud
        _same(_run(seq, "prefetch", deskew, depth=depth), want, ("prefetch", depth))
    _same(_run(seq, "prefetch_f32", deskew, depth=5), want, "prefetch_f32")


@gpu
def test_device_form_waits_for_the_consumer(built):
    import torch
    p = _pipeline()
    for i, a in enumerate(_sequence(4)):
        p.computeRecords(0.1 * i, a, **KITTI_GATE)
    want, want_idx = p.currentCloudArray(), p.currentCloudIndices()
    n = want.shape[0]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        junk = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        junk_i = torch.empty(n, dtype=torch.int64, device="cuda")
        torch.cuda._sleep(200_000_000)
        junk.fill_(float("nan"))  # behind the sleep, in memory the outputs are likely to reuse
        junk_i.fill_(-1)
        del junk, junk_i
        got = p.currentCloudArray(device=True)
        got_i = p.currentCloudIndices(device=True)
        copy, copy_i = got.clone(), got_i.clone()
    side.synchronize()
    assert got.dtype == torch.float64 and got_i.dtype == torch.int64
    assert bits_equal(got.cpu().numpy(), want) and bits_equal(copy.cpu().numpy(), want)
    assert (got_i.cpu().numpy() == want_idx).all() and (copy_i.cpu().numpy() == want_idx).all()
    assert bits_equal(p.currentCloudArray(device=True, frame="sensor").cpu().numpy(), p.currentCloudArray(frame="sensor"))
