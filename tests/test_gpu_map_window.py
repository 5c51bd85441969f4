"""The voxel map's window (madicp_map_remove_far, Pipeline(map_max_distance=D)).  A removal drops every voxel whose centre
(k + 0.5) v lies farther than D from an origin, ((dx dx + dy dy) + dz dz) > D^2 in float64 without FMA, with all its rows;
the rows that stay keep their order and (scan, record); a removed voxel is forgotten, so later points refill it.  The
oracle below restates that with numpy and is checked against a plain dict loop; every GPU comparison is bit for bit."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

from mad_icp_b200 import _capi, synth
from test_gpu_voxel_map import (CASES, KITTI_GATE, LIM, MapOracle, _edge_points, _iso_apply, _pipeline, _sequence,
                                raises_madicp)
from util import bits_equal

NEW_SYMBOLS = ["madicp_map_remove_far", "madicp_debug_map_table"]
INF = float("inf")
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- oracle
def _far(k, v, origin, D):
    """per row of integer-valued keys k (n, 3): the voxel's centre lies farther than D from origin"""
    c = (np.asarray(k, np.float64) + 0.5) * v
    d = c - np.asarray(origin, np.float64)
    return ((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) > np.float64(D) * np.float64(D)


class WindowOracle(MapOracle):
    """MapOracle plus remove_far; `removed` counts the voxels removed so far"""

    def __init__(self, v, K):
        super().__init__(v, K)
        self.removed = 0

    def remove_far(self, origin, D):
        if self.keys.size:
            f = (1 << 21) - 1
            k = np.column_stack([self.keys & f, (self.keys >> 21) & f, self.keys >> 42]) - LIM
            keep = ~_far(k, self.v, origin, D)
            self.removed += int((~keep).sum())
            self.keys, self.counts = self.keys[keep], self.counts[keep]
        xyz, sr = self.points()
        keep = ~_far(np.floor(xyz / self.v), self.v, origin, D)
        self.xyz, self.sr = [xyz[keep]], [sr[keep]]


def dict_window_oracle(ops, v, K):
    """the same point by point: ops are ("insert", P, scan, rec) and ("remove", origin, D)"""
    count, rows, dropped = {}, [], 0

    def far(key, origin, D):
        d = [(float(k) + 0.5) * v - o for k, o in zip(key, origin)]
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] > D * D

    for op in ops:
        if op[0] == "remove":
            _, origin, D = op
            origin = [float(o) for o in origin]
            count = {k: c for k, c in count.items() if not far(k, origin, D)}
            rows = [r for r in rows if not far(r[0], origin, D)]
            continue
        _, P, scan, rec = op
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
                rows.append((key, p, (scan, r)))
    xyz = np.array([r[1] for r in rows], np.float64).reshape(-1, 3)
    sr = np.array([r[2] for r in rows], np.int64).reshape(-1, 2)
    return xyz, sr, dropped, len(count)


def _ops(v, seed):
    """inserts of edge points (negative coordinates, -0.0, voxel boundaries, keys at +-(2^20 - 1), NaN, inf) between
    removals: a centre exactly at distance D (a tie, which stays), D = 0 around a voxel centre, D = inf, an origin next
    to the far keys, an origin far away (everything goes), and inserts that refill removed voxels"""
    rs = np.random.RandomState(seed)
    c0 = np.array([0.5, 0.5, 0.5]) * v  # the centre of voxel (0, 0, 0)
    removals = [(c0, 3 * v), (c0, 0.0), (c0, INF), (np.array([(LIM - 1.5) * v, 0.0, 0.0]), 4 * v), (c0, 5.5 * v),
                (np.array([1e6, -1e6, 3e5]), 1.0), (-c0, 2.25 * v)]
    ops = []
    for s, rem in enumerate(removals):
        P = _edge_points(v, 200, seed=100 * seed + s)
        P[:20] = (LIM - 1) * v + rs.rand(20, 3) * 0.5 * v  # near the key limit, where the fourth origin sits
        P[20:30] = P[30:40]  # repeats: voxels at K
        ops.append(("insert", P, s, np.arange(P.shape[0]) * 2 + s))
        ops.append(("remove", rem[0], float(rem[1])))
    P = _edge_points(v, 200, seed=999 + seed)  # refills after everything went
    ops.append(("insert", P, 50, np.arange(P.shape[0])))
    ops.append(("remove", c0, 4 * v))
    return ops


def _apply(o, ops):
    for op in ops:
        if op[0] == "insert":
            o.insert(*op[1:])
        else:
            o.remove_far(*op[1:])


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_symbols_bound_and_abi_unchanged(built):
    L = _capi.lib()
    for name in NEW_SYMBOLS:
        assert name in _capi.SYMBOLS and getattr(L, name).restype is not None
    assert L.madicp_abi_version() == 3


def test_bad_arguments_without_gpu(built):
    L = _capi.lib()
    fake = C.c_void_p(1)  # never dereferenced: the value checks come first
    o = np.zeros(3)
    assert L.madicp_map_remove_far(None, _capi.as_d(o), 1.0) < 0
    assert b"null map" in L.madicp_last_error()
    assert L.madicp_map_remove_far(fake, None, 1.0) < 0
    assert b"origin" in L.madicp_last_error()
    for D in (float("nan"), -1.0, -1e-300, -INF):
        assert L.madicp_map_remove_far(fake, _capi.as_d(o), D) < 0, D
        assert b"max_distance" in L.madicp_last_error()
    for a in range(3):
        for bad in (float("nan"), INF, -INF):
            x = np.zeros(3)
            x[a] = bad
            assert L.madicp_map_remove_far(fake, _capi.as_d(x), 1.0) < 0, (a, bad)
            assert b"origin" in L.madicp_last_error()
    assert L.madicp_debug_map_table(None, None, None, None) < 0


@pytest.mark.parametrize("v,K", [(0.25, 1), (0.25, 3), (1.0, 2), (0.1, 32)])
def test_numpy_oracle_is_the_dict_loop(v, K):
    for seed in range(2):
        ops = _ops(v, seed)
        o = WindowOracle(v, K)
        _apply(o, ops)
        xyz, sr = o.points()
        want_xyz, want_sr, dropped, live = dict_window_oracle(ops, v, K)
        assert bits_equal(xyz, want_xyz) and (sr == want_sr).all() and o.dropped == dropped
        assert o.keys.size == live and want_xyz.shape[0] > 0

    # the edges are reached (at a voxel size where the centres are exact): a tie at distance D stays, D = 0 keeps the
    # voxel whose centre is the origin, D = inf keeps all, a far origin takes all
    v = 0.25
    c0 = np.array([0.5, 0.5, 0.5]) * v
    o = WindowOracle(v, K)
    o.insert(np.array([[3.2 * v, 0.2 * v, 0.4 * v], [4.2 * v, 0.1 * v, 0.1 * v], [0.1 * v, -0.0, 0.9 * v]]), 0,
             np.arange(3))
    o.remove_far(c0, 3 * v)  # voxel (3, 0, 0): centre at exactly 3 v
    assert o.points()[1][:, 1].tolist() == [0, 2]
    o.remove_far(c0, 0.0)
    assert o.points()[1][:, 1].tolist() == [2]
    o.insert(np.array([[3.2 * v, 0.2 * v, 0.4 * v]]), 1, [7])  # the removed voxel starts afresh
    o.remove_far(c0, INF)
    assert o.points()[1].tolist() == [[0, 2], [1, 7]]
    o.remove_far(np.array([1e9, 0.0, 0.0]), 10.0)
    assert o.points()[0].shape == (0, 3) and o.keys.size == 0


# ----------------------------------------------------------------------------------------------------------- GPU
@pytest.fixture(scope="module")
def drive(built):
    """a Registrar keeping clouds and device trees of street scans along x, with out-of-range and NaN points"""
    from mad_icp_b200 import Registrar
    reg = Registrar(device=0, max_keyframes=4)
    reg.keep_cloud(True)
    scene = synth.StreetScene(seed=5, x_min=-45.0, x_max=90.0)
    trees, clouds, poses = [], [], []
    for i in range(6):
        P = synth.lidar_scan(scene, synth.pose_xyyaw(0.0, 0.5, 0.0), beams=32, azimuths=1024, seed=40 + i)
        rs = np.random.RandomState(i)
        bad = rs.choice(P.shape[0], 20, replace=False)
        P[bad[:10]] += np.array([3.0e6, 0.0, 0.0])
        P[bad[10:], 2] = np.nan
        trees.append(reg.build_tree(P))
        clouds.append(P)
        poses.append(synth.pose_xyyaw(6.0 * i, 0.3 * np.sin(i), 0.1 * i, z=0.05 * i))
    return reg, trees, clouds, poses


def _check(m, o, what):
    want_xyz, want_sr = o.points()
    assert m.size() == want_xyz.shape[0], what
    assert m.dropped() == o.dropped, what
    xyz, sr = m.points()
    assert bits_equal(xyz, want_xyz) and (sr == want_sr).all(), what


@gpu
@pytest.mark.parametrize("v,K,D", [(0.2, 1, 12.0), (0.5, 4, 8.0), (0.1, 32, 15.0), (0.2, 2, 0.0), (0.3, 3, INF)])
def test_engine_window_is_the_oracle(drive, v, K, D):
    reg, trees, clouds, poses = drive
    m = reg.voxel_map(v, K)  # reserve_points = 0: the map grows between removals
    o = WindowOracle(v, K)
    plain = reg.voxel_map(v, K)
    for s, (t, P, T) in enumerate(zip(trees, clouds, poses)):
        m.insert(t, T, scan=s)
        plain.insert(t, T, scan=s)
        o.insert(_iso_apply(T, P), s, np.arange(P.shape[0]))
        origin = np.asarray(T)[:3, 3]
        m.remove_far(origin, D)
        o.remove_far(origin, D)
        _check(m, o, (s, "window"))
    if D == INF:  # nothing goes: the same rows as the inserts alone
        xyz, sr = plain.points()
        assert bits_equal(m.points()[0], xyz) and (m.points()[1] == sr).all()
    else:
        assert o.removed > 0
    # an origin far away: everything goes; then the same trees refill the map from nothing
    m.remove_far([5.0e4, -3.0e4, 0.0], 100.0)
    o.remove_far([5.0e4, -3.0e4, 0.0], 100.0)
    _check(m, o, "far origin")
    assert m.size() == 0 and m.table()[2] == 0
    for s in (2, 3):
        m.insert(trees[s], poses[s], scan=100 + s)
        o.insert(_iso_apply(poses[s], clouds[s]), 100 + s, np.arange(clouds[s].shape[0]))
    m.remove_far(np.asarray(poses[3])[:3, 3], D)
    o.remove_far(np.asarray(poses[3])[:3, 3], D)
    _check(m, o, "refill")
    dx, ds = m.points(device=True)
    want_xyz, want_sr = o.points()
    assert bits_equal(dx.cpu().numpy(), want_xyz) and (ds.cpu().numpy() == want_sr).all()
    slots, occupied, live = m.table()
    assert live == o.keys.size and 2 * occupied <= slots
    m.clear()  # after removals: an empty map, then a fresh one
    assert m.size() == 0 and m.dropped() == 0 and m.table()[1] == 0
    m.insert(trees[1], poses[1], scan=7)
    o = WindowOracle(v, K)
    o.insert(_iso_apply(poses[1], clouds[1]), 7, np.arange(clouds[1].shape[0]))
    _check(m, o, "after clear")


def _churn_cloud(i, n, step):
    """n points in a 30 x 30 x 2 m box whose centre moves `step` m along x per scan"""
    rs = np.random.RandomState(1000 + i)
    return rs.uniform([-15.0, -15.0, -1.0], [15.0, 15.0, 1.0], size=(n, 3)) + np.array([step * i, 0.0, 0.0])


@gpu
def test_churn_keeps_the_table_bounded(drive):
    reg = drive[0]
    v, K, D, n, step, scans = 0.5, 2, 14.0, 6000, 3.0, 240
    m = reg.voxel_map(v, K)
    o = WindowOracle(v, K)
    created, peak_live, slots_seen = 0, 0, []
    for i in range(scans):
        P = _churn_cloud(i, n, step)
        t = reg.build_tree(P)
        before = set(o.keys.tolist())
        m.insert(t, None, scan=i)
        o.insert(P, i, np.arange(n))
        created += len(set(o.keys.tolist()) - before)
        origin = np.array([step * i, 0.0, 0.0])
        m.remove_far(origin, D)
        o.remove_far(origin, D)
        peak_live = max(peak_live, o.keys.size)
        if i % 20 == 19:
            slots, occupied, live = m.table()
            assert live == o.keys.size and 2 * occupied <= slots, i
            slots_seen.append(slots)
            _check(m, o, i)
    # many times more voxels went through the map than its table holds, and the table stayed within the policy's bound:
    # a rebuild leaves at most a quarter of the slots to live voxels and the points of one insert
    assert created >= 4 * max(slots_seen), (created, slots_seen)
    assert max(slots_seen) <= 8 * (peak_live + n), (slots_seen, peak_live)
    assert slots_seen[len(slots_seen) // 2:] == [slots_seen[-1]] * (len(slots_seen) - len(slots_seen) // 2)
    _check(m, o, "end")


# ----------------------------------------------------------------------------------------------------------- pipeline
@functools.lru_cache(maxsize=None)
def _seq(layout):
    return _sequence(40, layout)


def _run_window(case, deskew, lookahead, D):
    """a window pipeline and a plain one (no map) over the case's sequence; checks the map against the oracle after every
    scan, and the poses against the plain pipeline's"""
    layout, gate, field, scale, mkw = CASES[case]
    seq = _seq(layout)
    tkw = dict(time_field=field, time_scale=scale) if deskew == "time" else {}
    p = _pipeline(deskew=deskew != "none", keep=True, map_max_distance=D, **mkw)
    ref = _pipeline(deskew=deskew != "none", keep=False)
    o = WindowOracle(mkw["map_voxel_size"], mkw["map_points_per_voxel"])
    queued = 0
    for i, a in enumerate(seq):
        if lookahead:
            while queued < min(i + 4, len(seq)):
                assert p.prefetchRecords(seq[queued], **gate, deskew_ahead=deskew != "none", **tkw)
                queued += 1
        scan = p.currentID()
        p.computeRecords(0.1 * i, a, **gate, **tkw)
        ref.computeRecords(0.1 * i, a, **gate, **tkw)
        o.insert(p.currentCloudArray(frame="map"), scan, p.currentCloudIndices())
        o.remove_far(p.currentPose()[:3, 3], D)
        assert bits_equal(p.currentPose(), ref.currentPose()), i  # registration is untouched
        assert p.keyframeID() == ref.keyframeID() and p.inliersRatio() == ref.inliersRatio(), i
        if i % 8 == 7:
            assert bits_equal(p.mapArray(), o.points()[0]) and (p.mapIndices() == o.points()[1]).all(), i
    return p, o


@gpu
@pytest.mark.parametrize("lookahead", [False, True])
@pytest.mark.parametrize("deskew", ["none", "azimuth", "time"])
@pytest.mark.parametrize("case", ["kitti", "ouster"])
def test_pipeline_window_is_the_oracle(built, case, deskew, lookahead):
    D = 12.0
    p, o = _run_window(case, deskew, lookahead, D)
    want_xyz, want_sr = o.points()
    assert p.mapSize() == want_xyz.shape[0] > 0 and p.mapDropped() == o.dropped
    assert bits_equal(p.mapArray(), want_xyz) and (p.mapIndices() == want_sr).all()
    assert bits_equal(p.mapArray(device=True).cpu().numpy(), want_xyz)
    assert (p.mapIndices(device=True).cpu().numpy() == want_sr).all()
    # the drive went well past D, and no row lies farther from the last origin than D plus half a voxel diagonal
    v = CASES[case][4]["map_voxel_size"]
    assert o.removed > 0 and np.linalg.norm(p.currentPose()[:3, 3]) > 2 * D
    assert (np.linalg.norm(want_xyz - p.currentPose()[:3, 3], axis=1) <= D + v * np.sqrt(3) / 2 + 1e-9).all()


@gpu
def test_launches_and_clear(built):
    seq = _seq("kitti")[:10]
    mkw = dict(map_voxel_size=0.3, map_points_per_voxel=3)
    plain = _pipeline(deskew=True, keep=False, **mkw)
    zero = _pipeline(deskew=True, keep=False, map_max_distance=0.0, **mkw)
    wide = _pipeline(deskew=True, keep=False, map_max_distance=1.0e4, **mkw)  # removes nothing: rows and table as plain
    for i, a in enumerate(seq):
        for p in (plain, zero, wide):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
    assert zero._kernelLaunches() == plain._kernelLaunches()
    assert wide._kernelLaunches() - plain._kernelLaunches() == 5 * len(seq)  # 5 launches per removal
    assert bits_equal(wide.mapArray(), plain.mapArray())
    # clearMap after removals, then more scans: a fresh oracle's map
    p = _pipeline(deskew=True, keep=True, map_max_distance=6.0, **mkw)
    o = WindowOracle(0.3, 3)
    for i, a in enumerate(_seq("kitti")[:24]):
        if i == 14:
            p.clearMap()
            assert p.mapSize() == 0 and p.mapArray().shape == (0, 3)
            o = WindowOracle(0.3, 3)
        scan = p.currentID()
        p.computeRecords(0.1 * i, a, **KITTI_GATE)
        o.insert(p.currentCloudArray(frame="map"), scan, p.currentCloudIndices())
        o.remove_far(p.currentPose()[:3, 3], 6.0)
    assert o.removed > 0
    assert bits_equal(p.mapArray(), o.points()[0]) and (p.mapIndices() == o.points()[1]).all()


@gpu
def test_pipeline_rejects_a_bad_window(built):
    for bad in (dict(map_voxel_size=0.2, map_max_distance=-1.0), dict(map_voxel_size=0.2, map_max_distance=float("nan")),
                dict(map_voxel_size=0.2, map_max_distance=INF), dict(map_max_distance=10.0)):
        with raises_madicp("map_max_distance"):
            _pipeline(**bad)
