"""Nearest-row queries of the voxel map (madicp_map_nearest[_dev], VoxelMap.nearest, Pipeline.mapNearest).  For a query
q, the candidates are the map's rows whose scan is < scan_below; d2_j = ((x_j - qx)^2 + (y_j - qy)^2) + (z_j - qz)^2 in
float64 without FMA, r2 = max_distance^2; the answer is the candidate with the least d2_j among those with d2_j <= r2,
ties to the smallest row, or (-1, +inf).  The oracles below restate that by brute force and through a KD-tree at a
slightly larger radius (then the exact formula and the tie rule), and are checked against a plain Python loop; every
GPU comparison is bit for bit."""
import ctypes as C
import functools

import numpy as np
import pytest
from scipy.spatial import cKDTree

from mad_icp_b200 import _capi, synth
from test_gpu_map_window import WindowOracle, _churn_cloud, drive  # noqa: F401  (drive: a module fixture)
from test_gpu_voxel_map import CASES, LIM, MapOracle, _edge_points, _iso_apply, _pipeline, _sequence
from util import bits_equal

NEW_SYMBOLS = ["madicp_map_nearest", "madicp_map_nearest_dev"]
INF = float("inf")
NO_LIMIT = np.iinfo(np.int64).max
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- oracles
def _cands(sr, scan_below):
    return np.arange(sr.shape[0]) if scan_below is None else np.flatnonzero(sr[:, 0] < scan_below)


def nearest_brute(xyz, sr, Q, r, scan_below=None, chunk=128):
    """every (query, candidate) pair, in chunks of queries"""
    Q = np.asarray(Q, np.float64)
    row, d2 = np.full(Q.shape[0], -1, np.int64), np.full(Q.shape[0], INF)
    cand = _cands(sr, scan_below)
    if cand.size == 0:
        return row, d2
    P, r2 = xyz[cand], np.float64(r) * np.float64(r)
    for s in range(0, Q.shape[0], chunk):
        q = Q[s:s + chunk]
        with np.errstate(invalid="ignore", over="ignore"):
            d = P[None, :, :] - q[:, None, :]
            D = (d[:, :, 0] * d[:, :, 0] + d[:, :, 1] * d[:, :, 1]) + d[:, :, 2] * d[:, :, 2]
        ok = D <= r2
        j = np.argmin(np.where(ok, D, INF), axis=1)  # (the first of equal minima: the smallest row)
        hit = ok[np.arange(q.shape[0]), j]
        row[s:s + chunk][hit] = cand[j[hit]]
        d2[s:s + chunk][hit] = D[np.arange(q.shape[0]), j][hit]
    return row, d2


def nearest_oracle(xyz, sr, Q, r, scan_below=None, chunk=16384):
    """cKDTree.query_ball_point at a radius enlarged by 1e-9 relative (and 1e-150 for squares that underflow), then the
    exact formula, d2 <= r2 and the lexicographic (d2, row) minimum"""
    Q = np.asarray(Q, np.float64)
    row, d2 = np.full(Q.shape[0], -1, np.int64), np.full(Q.shape[0], INF)
    cand = _cands(sr, scan_below)
    if cand.size == 0:
        return row, d2
    P, r2 = xyz[cand], np.float64(r) * np.float64(r)
    with np.errstate(invalid="ignore"):  # (finite queries within the rows' bounding box grown by 2 r + 1e-6; the others
        pad = 2 * r + 1e-6              # are farther than r from every row, and overflow the KD-tree's distances)
        ok = np.flatnonzero(np.isfinite(Q).all(axis=1) & (Q >= P.min(axis=0) - pad).all(axis=1) &
                            (Q <= P.max(axis=0) + pad).all(axis=1))
    if ok.size == 0:
        return row, d2
    tree = cKDTree(P)
    for s in range(0, ok.size, chunk):
        qi = ok[s:s + chunk]
        lists = tree.query_ball_point(Q[qi], r * (1 + 1e-9) + 1e-150)
        lens = np.fromiter((len(x) for x in lists), np.int64, qi.size)
        if lens.sum() == 0:
            continue
        J = np.concatenate([np.asarray(x, np.int64) for x in lists if len(x)])
        I = np.repeat(qi, lens)
        d = P[J] - Q[I]
        D = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        keep = D <= r2
        I, J, D = I[keep], cand[J[keep]], D[keep]
        o = np.lexsort((J, D, I))
        I, J, D = I[o], J[o], D[o]
        first = np.ones(I.size, bool)
        first[1:] = I[1:] != I[:-1]
        row[I[first]], d2[I[first]] = J[first], D[first]
    return row, d2


def nearest_loop(xyz, sr, Q, r, scan_below=None):
    """the contract point by point, with Python floats"""
    r2 = float(r) * float(r)
    rows, d2s = [], []
    for q in Q:
        qx, qy, qz = (float(c) for c in q)
        best, bd = -1, INF
        for j, (p, t) in enumerate(zip(xyz, sr)):
            if scan_below is not None and int(t[0]) >= scan_below:
                continue
            dx, dy, dz = float(p[0]) - qx, float(p[1]) - qy, float(p[2]) - qz
            d = (dx * dx + dy * dy) + dz * dz
            if d <= r2 and (d < bd or (d == bd and j < best)):
                best, bd = j, d
        rows.append(best)
        d2s.append(bd)
    return np.array(rows, np.int64), np.array(d2s, np.float64)


def _same(got, want, what=""):
    row, d2 = (np.asarray(x.cpu() if hasattr(x, "cpu") else x) for x in got)
    assert (row == want[0]).all(), (what, np.flatnonzero(row != want[0])[:5])
    assert bits_equal(d2, want[1]), what


def _edge_case(v):
    """map rows from edge points (voxel boundaries, negative coordinates, -0.0, keys next to +-2^20) with a tie and a
    row at exactly r from a query, and queries among them, next to them, non-finite, at the key limit and at 1e300"""
    o = MapOracle(v, 3)
    o.insert(_edge_points(v, 300, seed=1), 4, np.arange(300))
    o.insert(np.array([[2.0, 0.0, 0.0], [0.0, 0.0, 0.0], [5.0, 5.0, 5.0], [5.0, 5.5, 5.0]]) * v * 4, 7, np.arange(4))
    o.insert(_edge_points(v, 300, seed=2), 9, np.arange(300))
    xyz, sr = o.points()
    rs = np.random.RandomState(3)
    Q = np.concatenate([xyz[rs.choice(xyz.shape[0], 40)],                               # on rows (r = 0 finds them)
                        xyz[rs.choice(xyz.shape[0], 40)] + rs.choice([-0.5, 0.25, 0.5, 0.0], (40, 3)) * v,
                        np.array([[1.0, 0.0, 0.0], [5.0, 5.25, 5.0]]) * v * 4,          # midpoints: ties
                        _edge_points(v, 60, seed=4),                                    # NaN, inf, key limit, -0.0
                        np.array([[1e300, 0.0, 0.0], [-1e300, -1e300, 1e300], [(LIM - 1) * v] * 3, [-LIM * v] * 3,
                                  [np.nan, 0.0, 0.0], [0.0, np.inf, 0.0], [-0.0, -0.0, -0.0]])])
    return xyz, sr, Q


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_symbols_bound_and_abi_unchanged(built):
    L = _capi.lib()
    for name in NEW_SYMBOLS:
        assert name in _capi.SYMBOLS and getattr(L, name).restype is not None
    assert L.madicp_abi_version() == 3


def test_bad_arguments_without_gpu(built):
    L = _capi.lib()
    fake = C.c_void_p(1)  # never dereferenced: the value checks come first
    q = np.zeros((4, 3))
    row, d2 = np.empty(4, np.int64), np.empty(4)
    rp = row.ctypes.data_as(C.POINTER(C.c_int64))
    host = lambda m, qq, n, r, rr, dd: L.madicp_map_nearest(m, qq, n, r, NO_LIMIT, rr, dd)  # noqa: E731
    dev = lambda m, qq, n, r, rr, dd: L.madicp_map_nearest_dev(m, qq, n, 24, 0, r, NO_LIMIT, rr, dd, None)  # noqa: E731
    for f in (host, dev):
        assert f(None, _capi.as_d(q), 4, 0.1, rp, _capi.as_d(d2)) < 0
        assert b"null map" in L.madicp_last_error()
        assert f(fake, _capi.as_d(q), -1, 0.1, rp, _capi.as_d(d2)) < 0
        assert b"n must be" in L.madicp_last_error()
        assert f(fake, _capi.as_d(q), 4, 0.1, None, None) < 0
        assert b"no output" in L.madicp_last_error()
        assert f(fake, None, 4, 0.1, rp, _capi.as_d(d2)) < 0
        assert b"null queries" in L.madicp_last_error()
        for r in (float("nan"), INF, -INF, -1.0, -1e-300):
            assert f(fake, _capi.as_d(q), 4, r, rp, _capi.as_d(d2)) < 0, r
            assert b"max_distance" in L.madicp_last_error()
    for stride, f32 in ((16, 0), (12, 0), (28, 0), (8, 1), (14, 1)):
        assert L.madicp_map_nearest_dev(fake, _capi.as_d(q), 4, stride, f32, 0.1, NO_LIMIT, rp, None, None) < 0
        assert b"stride" in L.madicp_last_error()


@pytest.mark.parametrize("v", [0.25, 0.1])
def test_oracles_are_the_loop(v):
    xyz, sr, Q = _edge_case(v)
    hits = 0
    for r in (0.0, 0.5 * v, v, 4 * v):
        for below in (None, 8, 5, 0):
            want = nearest_loop(xyz, sr, Q, r, below)
            _same(nearest_brute(xyz, sr, Q, r, below), want, (r, below))
            _same(nearest_oracle(xyz, sr, Q, r, below), want, (r, below))
            hits += int((want[0] >= 0).sum())
            if below == 0:
                assert (want[0] == -1).all()
    assert hits > 0
    # the edges are reached (v = 0.25: coordinates exact): a tie goes to the smaller row, a row at exactly r is kept,
    # r = 0 finds exact coincidences only, non-finite queries find nothing, nor does an empty map
    if v == 0.25:
        i0 = int(np.flatnonzero((xyz == [2.0, 0.0, 0.0]).all(axis=1))[0])
        i1 = int(np.flatnonzero((xyz == [0.0, 0.0, 0.0]).all(axis=1))[0])
        for pair in ([i0, i1], [i1, i0]):
            row, d2 = nearest_loop(xyz[pair], sr[pair], np.array([[1.0, 0.0, 0.0]]), 1.0)
            assert row[0] == 0 and d2[0] == 1.0
        row, d2 = nearest_loop(xyz[[i0]], sr[[i0]], np.array([[1.0, 0.0, 0.0]]), 1.0)
        assert row[0] == 0 and d2[0] == 1.0  # d2 == r2: kept
        row, d2 = nearest_loop(xyz[[i0]], sr[[i0]], np.array([[1.0, 0.0, 0.0]]), 0.9999)
        assert row[0] == -1 and d2[0] == INF
    row, _ = nearest_loop(xyz, sr, Q, 0.0)
    assert (row[:40] >= 0).all()
    bad = ~np.isfinite(Q).all(axis=1)
    assert bad.any() and (nearest_oracle(xyz, sr, Q, 4 * v)[0][bad] == -1).all()
    empty = nearest_oracle(np.empty((0, 3)), np.empty((0, 2), np.int64), Q, v)
    assert (empty[0] == -1).all() and np.isinf(empty[1]).all()


# ----------------------------------------------------------------------------------------------------------- GPU
def _queries(P, T, seed, n=1500, v=0.2):
    """n points of a posed cloud, half of them moved by up to 2 v, and the edge queries"""
    rs = np.random.RandomState(seed)
    X = _iso_apply(T, P[rs.choice(P.shape[0], n, replace=False)])
    X[: n // 2] += rs.uniform(-2 * v, 2 * v, size=(n // 2, 3))
    edge = np.array([[np.nan, 0.0, 0.0], [0.0, -np.inf, 0.0], [1e300, 1e300, 1e300], [-1e300, 0.0, 0.0],
                     [(LIM - 1) * v, 0.0, 0.0], [-0.0, -0.0, -0.0]])
    return np.concatenate([X, edge])


def _check_all(m, o, Q, v, what, scan_below=None, side=None):
    """the host form (float64) and the device form (float64 and float32, strided, produced on a side stream) against the
    oracle at r in {0, v/2, v, 4v}"""
    import torch
    side = side or torch.cuda.Stream()
    xyz, sr = o.points()
    with np.errstate(over="ignore"):
        Q32 = Q.astype(np.float32).astype(np.float64)
    for r in (0.0, 0.5 * v, v, 4 * v):
        want, want32 = nearest_oracle(xyz, sr, Q, r, scan_below), nearest_oracle(xyz, sr, Q32, r, scan_below)
        _same(m.nearest(Q, r, scan_below), want, (what, r, "host"))
        with torch.cuda.stream(side):  # the queries are written on the side stream, and answered there
            wide = torch.zeros((Q.shape[0], 5), dtype=torch.float64, device="cuda")
            wide[:, :3] = torch.from_numpy(Q).cuda(non_blocking=False)
            narrow = torch.zeros((Q.shape[0], 4), dtype=torch.float32, device="cuda")
            narrow[:, :3] = torch.from_numpy(Q32.astype(np.float32)).cuda()  # (exact: Q32 holds float32 values)
            got, got32 = m.nearest(wide[:, :3], r, scan_below), m.nearest(narrow[:, :3], r, scan_below)
            assert got[0].dtype == torch.int64 and got[1].dtype == torch.float64
        side.synchronize()
        _same(got, want, (what, r, "device f64"))
        _same(got32, want32, (what, r, "device f32"))
        if r == v and scan_below is None:
            assert (want[0] >= 0).any() or xyz.shape[0] == 0, what


@gpu
@pytest.mark.parametrize("v,K", [(0.2, 1), (0.5, 4), (0.1, 32)])
def test_engine_queries_interleaved(drive, v, K):  # noqa: F811
    import torch
    reg, trees, clouds, poses = drive
    side = torch.cuda.Stream()
    m = reg.voxel_map(v, K)
    o = WindowOracle(v, K)
    Q0 = _queries(clouds[0], poses[0], 0, v=v)
    _check_all(m, o, Q0, v, "empty map")
    for s, (t, P, T) in enumerate(zip(trees, clouds, poses)):
        m.insert(t, T, scan=s)
        o.insert(_iso_apply(T, P), s, np.arange(P.shape[0]))
        Q = _queries(clouds[(s + 1) % len(clouds)], poses[(s + 1) % len(poses)], s, v=v)
        _check_all(m, o, Q, v, (s, "insert"), scan_below=None if s % 2 else s, side=side)
        if s % 2:
            origin = np.asarray(T)[:3, 3]
            m.remove_far(origin, 10.0)
            o.remove_far(origin, 10.0)
            assert o.removed > 0
            _check_all(m, o, Q, v, (s, "removal"), scan_below=s - 1, side=side)
    xyz, sr = o.points()
    got = m.nearest(xyz[:500], 0.0)  # every row finds itself, or an equal row before it, at r = 0
    _same(got, nearest_oracle(xyz, sr, xyz[:500], 0.0), "rows at r = 0")
    assert (got[0] >= 0).all() and (got[0] <= np.arange(500)).all() and (got[1] == 0.0).all()
    row, d2 = m.nearest(xyz[:200], v, scan_below=-1)
    assert (row == -1).all() and np.isinf(d2).all()


@gpu
def test_stale_index_guard(drive):  # noqa: F811
    """a query after clear, growth, a table rebuild that drops tombstones, and a removal sees the map as it is then"""
    import torch
    reg, trees, clouds, poses = drive
    side = torch.cuda.Stream()
    v, K = 0.5, 2
    m = reg.voxel_map(v, K, 1)  # reserve 1 row: the first inserts grow the rows and the table
    o = WindowOracle(v, K)
    Q = _queries(clouds[1], poses[1], 7, v=v)
    for s in range(3):  # growth after each query
        m.insert(trees[s], poses[s], scan=s)
        o.insert(_iso_apply(poses[s], clouds[s]), s, np.arange(clouds[s].shape[0]))
        _check_all(m, o, Q, v, ("growth", s), side=side)
    m.clear()
    o = WindowOracle(v, K)
    _check_all(m, o, Q, v, "clear", side=side)
    assert (m.nearest(Q, v)[0] == -1).all()
    m.insert(trees[1], poses[1], scan=9)
    o.insert(_iso_apply(poses[1], clouds[1]), 9, np.arange(clouds[1].shape[0]))
    _check_all(m, o, Q, v, "after clear", side=side)
    # churn: removals leave tombstones until an insert rebuilds the table (fewer occupied slots afterwards)
    m, o = reg.voxel_map(v, K), WindowOracle(v, K)
    rebuilds, occupied = 0, 0
    for i in range(60):
        P = _churn_cloud(i, 6000, 3.0)
        Qc = np.concatenate([P[:400] + 0.1, _churn_cloud(i - 1, 400, 3.0)])
        m.insert(reg.build_tree(P), None, scan=i)
        o.insert(P, i, np.arange(P.shape[0]))
        slots, occ, live = m.table()
        if occ < occupied:
            rebuilds += 1
            _check_all(m, o, Qc, v, ("rebuild", i), side=side)
        elif i % 15 == 0:
            _check_all(m, o, Qc, v, ("insert", i), side=side)
        m.remove_far(np.array([3.0 * i, 0.0, 0.0]), 14.0)
        o.remove_far(np.array([3.0 * i, 0.0, 0.0]), 14.0)
        occupied = m.table()[1]
        if i % 10 == 9:
            _check_all(m, o, Qc, v, ("removal", i), side=side)
    assert rebuilds > 0 and o.removed > 0


@gpu
def test_launches(drive):  # noqa: F811
    import torch
    reg, trees, clouds, poses = drive
    m = reg.voxel_map(0.3, 3)
    m.insert(trees[0], poses[0], scan=0)
    Q = _queries(clouds[1], poses[1], 1, v=0.3)
    Qd = torch.from_numpy(Q).cuda()
    for form in (Q, Qd):
        l0 = reg.kernel_launches
        m.nearest(form, 0.3)  # the first query after a change: the index (3) and the query (1)
        l1 = reg.kernel_launches
        m.nearest(form, 0.6)
        m.nearest(form, 0.0, scan_below=0)
        l2 = reg.kernel_launches
        assert (l1 - l0, l2 - l1) == (4, 2), (l1 - l0, l2 - l1)
        m.insert(trees[1], poses[1], scan=1)
    m.remove_far(np.asarray(poses[1])[:3, 3], 10.0)
    l0 = reg.kernel_launches
    m.nearest(Q, 0.3)
    assert reg.kernel_launches - l0 == 4
    # a map that never had an insert: no index, one launch
    e = reg.voxel_map(0.3, 3)
    l0 = reg.kernel_launches
    row, d2 = e.nearest(Q, 0.3)
    assert reg.kernel_launches - l0 == 1 and (row == -1).all() and np.isinf(d2).all()
    assert e.nearest(np.empty((0, 3)), 0.3)[0].shape == (0,)
    # bad arguments that need the map
    L = _capi.lib()
    row, d2 = np.empty(Q.shape[0], np.int64), np.empty(Q.shape[0])
    for r in (4 * 0.3 * (1 + 1e-15), 10.0):
        assert L.madicp_map_nearest(m._h, _capi.as_d(Q), Q.shape[0], r, NO_LIMIT, row.ctypes.data_as(C.POINTER(C.c_int64)),
                                    _capi.as_d(d2)) < 0
        assert b"4 voxel sizes" in L.madicp_last_error()
    assert L.madicp_map_nearest_dev(m._h, C.c_void_p(Q.ctypes.data), Q.shape[0], 24, 0, 0.3, NO_LIMIT,
                                    C.c_void_p(row.ctypes.data), None, None) < 0
    assert b"device memory" in L.madicp_last_error()
    m.nearest(Q, 4 * 0.3)  # 4 v itself is accepted


# ----------------------------------------------------------------------------------------------------------- pipeline
@functools.lru_cache(maxsize=None)
def _seq(layout):
    return _sequence(40, layout)


@gpu
@pytest.mark.parametrize("lookahead,window", [(False, 0.0), (True, 12.0)])
@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("case", ["kitti", "ouster"])
def test_pipeline_queries_are_the_oracle(built, case, deskew, lookahead, window):
    import torch
    layout, gate, _, _, mkw = CASES[case]
    v = mkw["map_voxel_size"]
    seq = _seq(layout)
    p = _pipeline(deskew=deskew, keep=True, map_max_distance=window, **mkw)
    ref = _pipeline(deskew=deskew, keep=True, map_max_distance=window, **mkw)  # the same, never queried
    queued, hits = 0, {}
    for i, a in enumerate(seq):
        if lookahead:
            while queued < min(i + 4, len(seq)):
                assert p.prefetchRecords(seq[queued], **gate, deskew_ahead=deskew)
                assert ref.prefetchRecords(seq[queued], **gate, deskew_ahead=deskew)
                queued += 1
        scan = p.currentID()
        p.computeRecords(0.1 * i, a, **gate)
        ref.computeRecords(0.1 * i, a, **gate)
        r = (v, 0.5 * v, 4 * v, 0.0)[i % 4]
        xyz, sr = p.mapArray(), p.mapIndices()
        if i % 2:
            Q = p.currentCloudArray(frame="map", device=True)
            got = p.mapNearest(Q, r, scan_below=scan)
            Q = Q.cpu().numpy()
        else:
            Q = p.currentCloudArray(frame="map")
            got = p.mapNearest(Q, r, scan_below=scan)
        want = nearest_oracle(xyz, sr, Q, r, scan)
        _same(got, want, (i, r))
        hits[r] = hits.get(r, 0) + int((want[0] >= 0).sum())
        if i == len(seq) - 1:
            _same(p.mapNearest(Q, r), nearest_oracle(xyz, sr, Q, r), "no limit")
        assert bits_equal(p.currentPose(), ref.currentPose()), i  # registration is untouched
        assert p.keyframeID() == ref.keyframeID() and p.inliersRatio() == ref.inliersRatio(), i
    assert bits_equal(p.mapArray(), ref.mapArray())
    assert hits[4 * v] > 0 and hits[v] > 0  # the scans lie on what was mapped before them


@gpu
def test_pipeline_launches_and_no_map(built):
    from test_gpu_voxel_map import KITTI_GATE, raises_madicp
    seq = _seq("kitti")[:8]
    mkw = dict(map_voxel_size=0.3, map_points_per_voxel=3)
    plain = _pipeline(deskew=True, keep=True, **mkw)
    asks = _pipeline(deskew=True, keep=True, **mkw)
    for i, a in enumerate(seq):
        plain.computeRecords(0.1 * i, a, **KITTI_GATE)
        asks.computeRecords(0.1 * i, a, **KITTI_GATE)
        plain.currentCloudArray(device=True)
        Q = asks.currentCloudArray(device=True)
        asks.mapNearest(Q, 0.3)
        asks.mapNearest(Q, 0.6, scan_below=i)
    # a map never queried launches what it always did; each scan then costs the index (3) and two queries (1 each)
    assert asks._kernelLaunches() - plain._kernelLaunches() == 5 * len(seq)
    bare = _pipeline(deskew=True, keep=True)
    bare.computeRecords(0.0, seq[0], **KITTI_GATE)
    for pts in (bare.currentCloudArray(), bare.currentCloudArray(device=True)):
        with raises_madicp("builds no map"):
            bare.mapNearest(pts, 0.1)


@gpu
def test_scale_million_rows(built):
    """a map of more than a million rows, queried by a full 64 x 2048 scan"""
    import torch
    from mad_icp_b200 import Registrar
    reg = Registrar(device=0, max_keyframes=2)
    reg.keep_cloud(True)
    scene = synth.StreetScene(seed=11, x_min=-60.0, x_max=90.0)
    v, K = 0.1, 32
    m, o = reg.voxel_map(v, K), MapOracle(v, K)
    s = 0
    while sum(x.shape[0] for x in o.xyz) < 1_000_000:
        P = synth.lidar_scan(scene, synth.pose_xyyaw(1.0 * s, 0.0, 0.0), beams=64, azimuths=2048, seed=300 + s)
        T = synth.pose_xyyaw(1.0 * s, 0.02 * s, 0.01 * s)
        m.insert(reg.build_tree(P), T, scan=s)
        o.insert(_iso_apply(T, P), s, np.arange(P.shape[0]))
        s += 1
    xyz, sr = o.points()
    assert m.size() == xyz.shape[0] >= 1_000_000
    P = synth.lidar_scan(scene, synth.pose_xyyaw(2.5, 0.3, 0.0), beams=64, azimuths=2048, seed=999)
    Q = _iso_apply(synth.pose_xyyaw(2.5, 0.3, 0.05), P)
    assert Q.shape[0] >= 120_000
    for r in (0.5 * v, v):
        want = nearest_oracle(xyz, sr, Q, r)
        _same(m.nearest(Q, r), want, r)
        _same(m.nearest(torch.from_numpy(Q).cuda(), r), want, (r, "device"))
        assert (want[0] >= 0).mean() > 0.5
    want = nearest_oracle(xyz, sr, Q, v, scan_below=s // 2)
    _same(m.nearest(Q, v, scan_below=s // 2), want, "scan_below")
