"""The voxel map of every registered scan (Pipeline(map_voxel_size=v, map_points_per_voxel=K), madicp_map_*).  A voxel
(floor(p / v) per axis, |key| < 2^20) keeps the first K points that reach it: scans in insertion order, points in
kept-cloud order.  Rows are in acceptance order, each with (scan, record).  The oracle below restates that with numpy;
every comparison is bit for bit."""
import contextlib
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
NEW_SYMBOLS = ["madicp_map_create", "madicp_map_free", "madicp_map_insert", "madicp_map_size", "madicp_map_points",
               "madicp_map_points_dev", "madicp_map_clear"]
LIM = 2 ** 20
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- oracle
class MapOracle:
    """The map's contract in numpy: keys by np.floor(P / v), a per-voxel count, acceptance in point order."""

    def __init__(self, v, K):
        self.v, self.K = v, K
        self.keys = np.empty(0, np.int64)  # sorted
        self.counts = np.empty(0, np.int64)
        self.xyz, self.sr, self.dropped = [], [], 0

    def insert(self, P, scan, rec):
        with np.errstate(invalid="ignore", over="ignore"):
            k = np.floor(P / self.v)
        ok = ((k > -LIM) & (k < LIM)).all(axis=1)
        self.dropped += int((~ok).sum())
        idx = np.flatnonzero(ok)
        if idx.size == 0:
            return
        k = k[idx].astype(np.int64) + LIM
        key = k[:, 0] | (k[:, 1] << 21) | (k[:, 2] << 42)
        uniq, inv = np.unique(key, return_inverse=True)
        order = np.argsort(inv, kind="stable")
        first = np.searchsorted(inv[order], inv[order], side="left")
        rank = np.empty(idx.size, np.int64)
        rank[order] = np.arange(idx.size) - first
        pos = np.minimum(np.searchsorted(self.keys, uniq), max(self.keys.size - 1, 0))
        found = self.keys[pos] == uniq if self.keys.size else np.zeros(uniq.size, bool)
        prev = np.where(found, self.counts[pos], 0) if self.keys.size else np.zeros(uniq.size, np.int64)
        accept = prev[inv] + rank < self.K
        acc = idx[accept]
        self.xyz.append(P[acc])
        self.sr.append(np.column_stack([np.full(acc.size, scan, np.int64), np.asarray(rec, np.int64)[acc]]))
        new = prev + np.bincount(inv[accept], minlength=uniq.size)
        self.counts[pos[found]] = new[found]
        self.keys = np.concatenate([self.keys, uniq[~found]])
        self.counts = np.concatenate([self.counts, new[~found]])
        o = np.argsort(self.keys)
        self.keys, self.counts = self.keys[o], self.counts[o]

    def points(self):
        if not self.xyz:
            return np.empty((0, 3)), np.empty((0, 2), np.int64)
        return np.concatenate(self.xyz), np.concatenate(self.sr)


def dict_oracle(scans, v, K):
    """the same with a plain dict, point by point"""
    import math
    count, xyz, sr, dropped = {}, [], [], 0
    for P, scan, rec in scans:
        for p, r in zip(P, rec):
            try:
                key = tuple(math.floor(float(c) / v) for c in p)
            except (ValueError, OverflowError):  # NaN / inf
                dropped += 1
                continue
            if any(not -LIM < q < LIM for q in key):
                dropped += 1
                continue
            if count.get(key, 0) < K:
                count[key] = count.get(key, 0) + 1
                xyz.append(p)
                sr.append((scan, r))
    return np.array(xyz, np.float64).reshape(-1, 3), np.array(sr, np.int64).reshape(-1, 2), dropped


def _edge_points(v, n, seed):
    """negative coordinates, exact voxel boundaries, -0.0, keys just inside / outside +-2^20, NaN and inf"""
    rs = np.random.RandomState(seed)
    P = rs.randint(-8, 8, size=(n, 3)) * v + rs.choice([0.0, 0.5 * v, -1e-9], size=(n, 3))
    P[rs.rand(n) < 0.1, 0] = -0.0
    edge = np.array([(LIM - 1) * v, LIM * v, -(LIM - 1) * v, -LIM * v, -LIM * v + 1e-3 * v, np.nan, np.inf, -np.inf])
    rows = rs.randint(0, n, size=40)
    P[rows, rs.randint(0, 3, size=40)] = edge[rs.randint(0, edge.size, size=40)]
    return P


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_symbols_bound_and_abi_unchanged(built):
    L = _capi.lib()
    for name in NEW_SYMBOLS:
        assert name in _capi.SYMBOLS and getattr(L, name).restype is not None
    assert L.madicp_abi_version() == 3


def test_bad_arguments_without_gpu(built):
    L = _capi.lib()
    out = C.c_void_p()
    fake = C.c_void_p(1)  # never dereferenced: the value checks come first
    assert L.madicp_map_create(None, 0.2, 1, 0, C.byref(out)) < 0
    assert b"null context" in L.madicp_last_error()
    for v in (0.0, -0.2, float("nan"), float("inf")):
        assert L.madicp_map_create(fake, v, 1, 0, C.byref(out)) < 0, v
        assert b"voxel_size" in L.madicp_last_error()
    for K in (0, -1, 33):
        assert L.madicp_map_create(fake, 0.2, K, 0, C.byref(out)) < 0, K
        assert b"points_per_voxel" in L.madicp_last_error()
    assert L.madicp_map_create(fake, 0.2, 1, -1, C.byref(out)) < 0
    assert L.madicp_map_free(None) < 0
    assert L.madicp_map_insert(None, None, None, 0) < 0
    assert b"null map" in L.madicp_last_error()
    assert L.madicp_map_size(None, None) < 0
    xyz, sr = np.empty((4, 3)), np.empty((4, 2), np.int64)
    assert L.madicp_map_points(None, _capi.as_d(xyz), sr.ctypes.data_as(C.POINTER(C.c_int64))) < 0
    assert L.madicp_map_points_dev(None, None, None, None) < 0
    assert L.madicp_map_clear(None) < 0


@pytest.mark.parametrize("v,K", [(0.25, 1), (0.25, 3), (1.0, 2)])
def test_numpy_oracle_is_the_dict_loop(v, K):
    scans = []
    for s in range(4):
        P = _edge_points(v, 300, seed=s)
        scans.append((P, s, np.arange(P.shape[0]) * 3 + s))
    o = MapOracle(v, K)
    for P, s, rec in scans:
        o.insert(P, s, rec)
    xyz, sr = o.points()
    want_xyz, want_sr, dropped = dict_oracle(scans, v, K)
    assert bits_equal(xyz, want_xyz) and (sr == want_sr).all() and o.dropped == dropped
    assert dropped > 0 and (np.signbit(xyz) & (xyz == 0.0)).any()  # -0.0 kept as -0.0
    assert (np.abs(np.floor(xyz / v)) == LIM - 1).any()  # keys just inside the range are kept


# ----------------------------------------------------------------------------------------------------------- GPU
def _iso_apply(T, p):
    X = np.asarray(T, np.float64)[:3]
    return ((X[None, :, 0] * p[:, 0:1] + X[None, :, 1] * p[:, 1:2]) + X[None, :, 2] * p[:, 2:3]) + X[None, :, 3]


@pytest.fixture(scope="module")
def engine_clouds(built):
    """a Registrar keeping clouds, and three device trees of street scans with out-of-range and NaN points"""
    from mad_icp_b200 import Registrar
    reg = Registrar(device=0, max_keyframes=4)
    reg.keep_cloud(True)
    scene = synth.StreetScene(seed=3, x_min=-45.0, x_max=80.0)
    trees, clouds = [], []
    for i in range(3):
        P = synth.lidar_scan(scene, synth.pose_xyyaw(1.5 * i, 0.5, 0.05 * i), beams=32, azimuths=1024, seed=20 + i)
        rs = np.random.RandomState(i)
        far = rs.choice(P.shape[0], 30, replace=False)
        P[far[:10]] = P[far[:10]] + np.array([2.0e6, 0.0, 0.0])  # keys out of range at every voxel size
        P[far[10:20], 1] = -4.0e6
        P[far[20:], 2] = np.nan
        t = reg.build_tree(P)
        trees.append(t)
        clouds.append(P)
    return reg, trees, clouds


POSES = [None, synth.pose_xyyaw(3.0, -1.0, 0.4, z=0.2), synth.pose_xyyaw(-7.5, 2.0, -1.1, z=-0.3)]


def _engine_map(reg, trees, v, K, reserve=0, device=False):
    m = reg.voxel_map(v, K, reserve)
    for s, (t, T) in enumerate(zip(trees, POSES)):
        m.insert(t, T, scan=10 + s)
    xyz, sr = m.points(device=device)
    return m, xyz, sr


@gpu
@pytest.mark.parametrize("K", [1, 3, 32])
@pytest.mark.parametrize("v", [0.05, 0.2, 1.0])
def test_engine_map_is_the_oracle(engine_clouds, v, K):
    reg, trees, clouds = engine_clouds
    o = MapOracle(v, K)
    for s, (P, T) in enumerate(zip(clouds, POSES)):  # the host input, posed by numpy: record = row
        o.insert(P if T is None else _iso_apply(T, P), 10 + s, np.arange(P.shape[0]))
    want_xyz, want_sr = o.points()
    m, xyz, sr = _engine_map(reg, trees, v, K)
    assert m.size() == want_xyz.shape[0] and m.dropped() == o.dropped == 3 * 30
    assert bits_equal(xyz, want_xyz) and (sr == want_sr).all()
    assert np.isnan(np.concatenate(clouds)).any()
    # a map that starts at one row grows and rehashes many times: the same bits
    _, xyz1, sr1 = _engine_map(reg, trees, v, K, reserve=1)
    assert bits_equal(xyz1, want_xyz) and (sr1 == want_sr).all()
    _, xyz2, sr2 = _engine_map(reg, trees, v, K, reserve=1 << 20)
    assert bits_equal(xyz2, want_xyz) and (sr2 == want_sr).all()
    # again, and through the device form
    _, dx, ds = _engine_map(reg, trees, v, K, device=True)
    assert bits_equal(dx.cpu().numpy(), want_xyz) and (ds.cpu().numpy() == want_sr).all()
    m.clear()
    assert m.size() == 0 and m.dropped() == 0
    m.insert(trees[1], POSES[1], scan=5)
    o = MapOracle(v, K)
    o.insert(_iso_apply(POSES[1], clouds[1]), 5, np.arange(clouds[1].shape[0]))
    xyz, sr = m.points()
    assert bits_equal(xyz, o.points()[0]) and (sr == o.points()[1]).all()


@gpu
def test_engine_map_rejects_bad_trees(built, engine_clouds):
    from mad_icp_b200 import Registrar
    reg, trees, clouds = engine_clouds
    m = reg.voxel_map(0.2)
    other = Registrar(device=0, max_keyframes=2)
    other.keep_cloud(True)
    t_other = other.build_tree(clouds[0])
    L = _capi.lib()
    assert L.madicp_map_insert(m._h, t_other._h, None, 0) == -1  # MADICP_ERR_INVALID
    assert b"another context" in L.madicp_last_error()
    reg.keep_cloud(False)
    try:
        bare = reg.build_tree(clouds[0])
    finally:
        reg.keep_cloud(True)
    assert L.madicp_map_insert(m._h, bare._h, None, 0) == -3  # MADICP_ERR_STATE
    assert b"kept no cloud" in L.madicp_last_error()
    host = np.empty((4, 3))
    assert L.madicp_map_points_dev(m._h, C.c_void_p(host.ctypes.data), None, None) < 0
    assert b"device memory" in L.madicp_last_error()
    assert m.size() == 0
    del t_other
    other.close()


# ----------------------------------------------------------------------------------------------------------- pipeline
@contextlib.contextmanager
def raises_madicp(match):
    """A MadIcpError from a Pipeline call.  Every pybind module registers a MadIcpError for the library's error type and
    the one registered last is raised, whichever module the call came from: it is caught as the RuntimeError all of them
    derive from, and checked by name."""
    with pytest.raises(RuntimeError, match=match) as e:
        yield e
    assert e.type.__name__ == "MadIcpError", e.type


def _pipeline(deskew=True, keep=True, gpu_build=True, **map_kw):
    from mad_icp_b200.pybind.pypeline import Pipeline
    os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
    try:
        return Pipeline(sensor_hz=10.0, deskew=deskew, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02,
                        num_keyframes=4, num_threads=4, realtime=False, keep_cloud=keep, **map_kw)
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


def _kept(a, gate):
    mask = records.range_mask(a, **gate).astype(bool)
    return np.column_stack([a["x"], a["y"], a["z"]])[mask].astype(np.float64) if a.dtype.names else \
        np.asarray(a[:, :3])[mask].astype(np.float64), np.flatnonzero(mask)


CASES = {  # layout, gate, time field (deskew "time"), map settings
    "kitti": ("kitti", KITTI_GATE, 3, 1.0, dict(map_voxel_size=0.2, map_points_per_voxel=1)),
    "ouster": ("ouster", OUSTER_GATE, "t", 1e-9, dict(map_voxel_size=0.5, map_points_per_voxel=4)),
}


@gpu
@pytest.mark.parametrize("deskew", ["none", "azimuth", "time"])
@pytest.mark.parametrize("case", ["kitti", "ouster"])
def test_pipeline_map_is_the_oracle(built, case, deskew):
    layout, gate, field, scale, mkw = CASES[case]
    seq = _sequence(40, layout)
    kw = dict(time_field=field, time_scale=scale) if deskew == "time" else {}
    p = _pipeline(deskew=deskew != "none", **mkw)
    ref = _pipeline(deskew=deskew != "none", keep=False)
    o = MapOracle(mkw["map_voxel_size"], mkw["map_points_per_voxel"])
    for i, a in enumerate(seq):
        scan = p.currentID()
        p.computeRecords(0.1 * i, a, **gate, **kw)
        ref.computeRecords(0.1 * i, a, **gate, **kw)
        o.insert(p.currentCloudArray(frame="map"), scan, p.currentCloudIndices())
        assert bits_equal(p.currentPose(), ref.currentPose()), i  # registration is untouched
        assert p.keyframeID() == ref.keyframeID() and p.inliersRatio() == ref.inliersRatio(), i
        assert p.lastIcpIterations() == ref.lastIcpIterations()
    want_xyz, want_sr = o.points()
    assert p.mapSize() == want_xyz.shape[0] > 0 and p.mapDropped() == o.dropped
    assert bits_equal(p.mapArray(), want_xyz) and (p.mapIndices() == want_sr).all()
    assert bits_equal(p.mapArray(device=True).cpu().numpy(), want_xyz)
    assert (p.mapIndices(device=True).cpu().numpy() == want_sr).all()
    assert np.unique(want_sr[:, 0]).size == 40  # every scan contributed
    assert all(bits_equal(T, U) for T, U in zip(p.trajectory(), ref.trajectory()))


def _run(seq, mode, depth=0, shift=0, **kw):
    """a sequence through one ingest path; returns the map (xyz, (scan, record)) with packed rows mapped to records"""
    import torch
    p = _pipeline(deskew=False, keep=False, map_voxel_size=0.2, map_points_per_voxel=2, **kw)
    kept = [_kept(a, KITTI_GATE) for a in seq]
    queued = 0
    for i, a in enumerate(seq):
        if mode == "prefetch":
            while queued < min(i + depth, len(seq)):
                assert p.prefetchRecords(seq[queued], **KITTI_GATE)
                queued += 1
        if mode in ("records", "prefetch"):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
        elif mode == "cuda":
            raw = np.frombuffer(a.tobytes(), np.uint8)
            buf = torch.zeros(raw.size + 64, dtype=torch.uint8, device="cuda")
            buf[shift:shift + raw.size] = torch.from_numpy(raw.copy()).cuda()
            p.computeRecords(0.1 * i, buf[shift:shift + raw.size].view(torch.float32).view(-1, 4), **KITTI_GATE)
        elif mode == "f32":
            p.compute(0.1 * i, kept[i][0].astype(np.float32))
        elif mode == "f64":
            p.compute(0.1 * i, kept[i][0])
        elif mode == "vec":
            from mad_icp_b200.pybind.pypeline import VectorEigen3d
            p.compute(0.1 * i, VectorEigen3d(kept[i][0]))
    xyz, sr = p.mapArray(), p.mapIndices()
    if mode in ("f32", "f64", "vec"):  # a packed cloud's rows -> the records'
        sr = sr.copy()
        for s in range(len(seq)):
            rows = sr[:, 0] == s
            sr[rows, 1] = kept[s][1][sr[rows, 1]]
    return xyz, sr


@gpu
def test_same_map_on_every_ingest_path(built):
    seq = _sequence(30)
    want_xyz, want_sr = _run(seq, "records")
    assert want_xyz.shape[0] > 0

    def same(got, what):
        assert bits_equal(got[0], want_xyz) and (got[1] == want_sr).all(), what

    same(_run(seq, "records"), "again")
    for shift in (4, 8, 12):
        same(_run(seq, "cuda", shift=shift), ("cuda", shift))
    for depth in (1, 5, 32):
        same(_run(seq, "prefetch", depth=depth), ("prefetch", depth))
    for mode in ("f32", "f64", "vec"):
        same(_run(seq, mode), mode)


@gpu
def test_keep_cloud_off_and_clear(built):
    seq = _sequence(12)
    mkw = dict(map_voxel_size=0.3, map_points_per_voxel=3)
    p = _pipeline(deskew=True, keep=False, **mkw)
    q = _pipeline(deskew=True, keep=True, **mkw)
    o = MapOracle(0.3, 3)
    for i, a in enumerate(seq):
        if i == 6:
            p.clearMap()
            assert p.mapSize() == 0 and p.mapArray().shape == (0, 3)
        scan = q.currentID()
        p.computeRecords(0.1 * i, a, **KITTI_GATE)
        q.computeRecords(0.1 * i, a, **KITTI_GATE)
        if i >= 6:
            o.insert(q.currentCloudArray(), scan, q.currentCloudIndices())
    for call in (lambda: p.currentCloudArray(), lambda: p.currentCloudIndices(), lambda: p.currentCloudArray(device=True)):
        with raises_madicp("keep_cloud"):
            call()
    want_xyz, want_sr = o.points()
    assert bits_equal(p.mapArray(), want_xyz) and (p.mapIndices() == want_sr).all()
    assert q.mapSize() > p.mapSize()


@gpu
def test_device_form_waits_for_the_consumer(built):
    import torch
    p = _pipeline(deskew=False, map_voxel_size=0.2)
    for i, a in enumerate(_sequence(4)):
        p.computeRecords(0.1 * i, a, **KITTI_GATE)
    want, want_sr = p.mapArray(), p.mapIndices()
    n = want.shape[0]
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        junk = torch.empty((n, 3), dtype=torch.float64, device="cuda")
        junk_i = torch.empty((n, 2), dtype=torch.int64, device="cuda")
        torch.cuda._sleep(200_000_000)
        junk.fill_(float("nan"))  # behind the sleep, in memory the outputs are likely to reuse
        junk_i.fill_(-1)
        del junk, junk_i
        got = p.mapArray(device=True)
        got_i = p.mapIndices(device=True)
        copy, copy_i = got.clone(), got_i.clone()
    side.synchronize()
    assert got.dtype == torch.float64 and got_i.dtype == torch.int64 and tuple(got_i.shape) == (n, 2)
    assert bits_equal(got.cpu().numpy(), want) and bits_equal(copy.cpu().numpy(), want)
    assert (got_i.cpu().numpy() == want_sr).all() and (copy_i.cpu().numpy() == want_sr).all()


@gpu
def test_no_map_runs_nothing_new(built):
    from mad_icp_b200.pybind.pypeline import Pipeline
    seq = _sequence(8)
    a = _pipeline(deskew=True, keep=False)
    b = Pipeline(sensor_hz=10.0, deskew=True, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
                 num_threads=4, realtime=False)
    for i, s in enumerate(seq):
        a.computeRecords(0.1 * i, s, **KITTI_GATE)
        b.computeRecords(0.1 * i, s, **KITTI_GATE)
    assert a._kernelLaunches() == b._kernelLaunches()
    for call in (a.mapSize, a.mapArray, a.mapIndices, a.mapDropped, a.clearMap, lambda: a.mapArray(device=True)):
        with raises_madicp("map_voxel_size"):
            call()
    with raises_madicp("map"):
        _pipeline(gpu_build=False, map_voxel_size=0.2)
    for bad in (dict(map_voxel_size=-0.1), dict(map_voxel_size=float("nan")), dict(map_voxel_size=float("inf")),
                dict(map_voxel_size=0.2, map_points_per_voxel=0), dict(map_voxel_size=0.2, map_points_per_voxel=33),
                dict(map_points_per_voxel=40)):
        with raises_madicp("map_"):
            _pipeline(**bad)
    # with a map: the launches of the pipeline that keeps clouds, plus K + 3 per scan (and a rehash per table growth)
    k = _pipeline(deskew=True, keep=True)
    m = _pipeline(deskew=True, keep=False, map_voxel_size=0.2, map_points_per_voxel=2)
    for i, s in enumerate(seq):
        k.computeRecords(0.1 * i, s, **KITTI_GATE)
        m.computeRecords(0.1 * i, s, **KITTI_GATE)
    extra = m._kernelLaunches() - k._kernelLaunches()
    assert 5 * len(seq) <= extra <= 5 * len(seq) + 4
