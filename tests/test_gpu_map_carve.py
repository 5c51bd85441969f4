"""Carving the voxel map along a scan's rays (madicp_map_carve, VoxelMap.carve, Pipeline(map_carve=r)).  A ray runs from
the origin's cell a = key(o) to the endpoint's cell b = key(p), with the insert's keys; with d = b - a and n = max |d| it
visits a + floor_div(2 d t + n, 2 n) per axis, t = 0 .. n, and carves the steps with double(t) < RN(reach n).  Rays with
n == 0 or n > 16384 carve nothing, an endpoint without a key has no ray, an origin without one carves nothing.  Every
live voxel a carved step visits goes with its rows, unless it holds an endpoint of the call.  The oracle below restates
that with numpy and is checked against a plain dict loop; every GPU comparison is bit for bit."""
import ctypes as C
import functools
import math

import numpy as np
import pytest

from mad_icp_b200 import _capi, synth
from test_gpu_map_window import WindowOracle, _ops, dict_window_oracle  # noqa: F401  (dict_window_oracle: the same rules)
from test_gpu_voxel_map import CASES, KITTI_GATE, LIM, _edge_points, _iso_apply, _pipeline, _sequence, raises_madicp
from util import bits_equal

MAX_RAY = 16384
CARVE_LAUNCHES = 7  # mark, spare, slot pass, row pass, sums, compact, copy back
INF = float("inf")
gpu = pytest.mark.gpu


# ----------------------------------------------------------------------------------------------------------- oracle
def _cells(P, v):
    """integer keys (n, 3) of the points as the insert keys them, and which points have one"""
    with np.errstate(invalid="ignore", over="ignore"):
        k = np.floor(np.asarray(P, np.float64).reshape(-1, 3) / v)
    ok = ((k > -LIM) & (k < LIM)).all(axis=1)
    return np.where(ok[:, None], k, 0).astype(np.int64), ok


def _pack(k):
    k = np.asarray(k, np.int64) + LIM
    return k[:, 0] | (k[:, 1] << 21) | (k[:, 2] << 42)


def carve_sets(P, origin, v, reach, chunk=1 << 14):
    """(the packed keys the carved steps of the rays visit, the packed keys of the endpoints), both unique"""
    kb, ok = _cells(P, v)
    ends = np.unique(_pack(kb[ok]))
    ka, oka = _cells(origin, v)
    if not oka[0]:
        return np.empty(0, np.int64), ends
    d = kb[ok] - ka
    n = np.abs(d).max(axis=1)
    ray = (n > 0) & (n <= MAX_RAY)
    d, n = d[ray], n[ray]
    seen = []
    for s in range(0, n.size, chunk):  # every step t = 0 .. n of each ray, then the carved ones
        dc, nc = d[s:s + chunk], n[s:s + chunk]
        idx = np.repeat(np.arange(nc.size), nc + 1)
        t = np.arange(idx.size) - np.repeat(np.cumsum(nc + 1) - (nc + 1), nc + 1)
        carved = t.astype(np.float64) < np.float64(reach) * nc.astype(np.float64)[idx]
        idx, t = idx[carved], t[carved]
        k = ka + (2 * dc[idx] * t[:, None] + nc[idx, None]) // (2 * nc[idx, None])  # (numpy's // floors)
        seen.append(np.unique(_pack(k)))
    return (np.unique(np.concatenate(seen)) if seen else np.empty(0, np.int64)), ends


class CarveOracle(WindowOracle):
    """WindowOracle plus carve; `removed` counts the voxels removed so far, by windows and carves"""

    def carve(self, P, origin, reach):
        """P: the endpoints as the map stores them (posed); origin: the rays' origin"""
        visited, ends = carve_sets(P, origin, self.v, reach)
        gone = np.intersect1d(np.setdiff1d(visited, ends), self.keys)
        if gone.size == 0:
            return
        keep = ~np.isin(self.keys, gone)
        self.removed += int(gone.size)
        self.keys, self.counts = self.keys[keep], self.counts[keep]
        xyz, sr = self.points()
        keep = ~np.isin(_pack(_cells(xyz, self.v)[0]), gone)
        self.xyz, self.sr = [xyz[keep]], [sr[keep]]


def dict_carve_oracle(ops, v, K):
    """the same point by point and step by step: ops are ("insert", P, scan, rec), ("remove", origin, D) and
    ("carve", P, origin, reach)"""
    count, rows, dropped = {}, [], 0

    def key(p):
        try:
            k = tuple(math.floor(float(c) / v) for c in p)
        except (ValueError, OverflowError):  # NaN / inf
            return None
        return k if all(-LIM < q < LIM for q in k) else None

    def far(k, origin, D):
        d = [(float(q) + 0.5) * v - o for q, o in zip(k, origin)]
        return (d[0] * d[0] + d[1] * d[1]) + d[2] * d[2] > D * D

    for op in ops:
        if op[0] == "remove":
            origin, D = [float(o) for o in op[1]], op[2]
            count = {k: c for k, c in count.items() if not far(k, origin, D)}
            rows = [r for r in rows if not far(r[0], origin, D)]
        elif op[0] == "carve":
            _, P, origin, reach = op
            a = key(origin)
            if a is None:
                continue
            ends = {key(p) for p in P} - {None}
            gone = set()
            for b in (key(p) for p in P):
                if b is None:
                    continue
                d = [q - r for q, r in zip(b, a)]
                n = max(abs(q) for q in d)
                if n == 0 or n > MAX_RAY:
                    continue
                t = 0
                while float(t) < reach * float(n):
                    k = tuple(r + (2 * q * t + n) // (2 * n) for q, r in zip(d, a))
                    if k in count and k not in ends:
                        gone.add(k)
                    t += 1
            count = {k: c for k, c in count.items() if k not in gone}
            rows = [r for r in rows if r[0] not in gone]
        else:
            _, P, scan, rec = op
            for p, r in zip(P, rec):
                k = key(p)
                if k is None:
                    dropped += 1
                elif count.get(k, 0) < K:
                    count[k] = count.get(k, 0) + 1
                    rows.append((k, p, (scan, r)))
    xyz = np.array([r[1] for r in rows], np.float64).reshape(-1, 3)
    sr = np.array([r[2] for r in rows], np.int64).reshape(-1, 2)
    return xyz, sr, dropped, len(count)


def _centres(keys, v):
    return (np.asarray(keys, np.float64) + 0.5) * v


def _carve_ops(v, seed):
    """the window's edge ops, then carves over a block of filled voxels around cell 0: axis-aligned, diagonal and
    negative rays, floor_div half-way ties in both signs of d, n = 0, n = 16384 (carves) and 16385 (does not), NaN and inf
    endpoints, reach 1, a tiny reach and one where reach n is an exact integer, voxels at K, refills of carved voxels, an
    origin out of range and rays between keys at +-(2^20 - 1)"""
    rs = np.random.RandomState(seed)
    ops = list(_ops(v, seed))
    g = np.arange(-6, 7)
    block = _centres(np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3), v)
    line = _centres([[t, 0, 0] for t in (1, 2, 100, 8191, 16383, 16384, 16385)], v)
    edge = _centres([[LIM - 1 - t, 0, 0] for t in range(0, 120, 3)] + [[-(LIM - 1) + t, 0, 0] for t in range(0, 120, 3)]
                    + [[LIM - 1, LIM - 1, LIM - 1], [-(LIM - 1), -(LIM - 1), -(LIM - 1)]], v)
    fill = np.concatenate([block, block + 0.25 * v, line, edge])  # (every block voxel twice: at K for K <= 2)
    c0 = _centres([[0, 0, 0]], v)[0]

    def insert(s):
        ops.append(("insert", fill, 60 + s, np.arange(fill.shape[0])))

    rays = _centres([[5, 0, 0], [-5, 0, 0], [0, 5, 0], [0, -6, 0], [0, 0, -5], [4, 4, 4], [-3, -3, 3], [5, -5, -5],
                     [2, 1, 0], [2, -1, 0], [6, 3, -3], [6, -3, 3], [4, 1, -1], [-4, -1, 1], [0, 6, 3], [0, 0, 0],
                     [16385, 0, 0]], v)
    bad = np.array([[np.nan, 0.0, 0.0], [0.0, np.inf, 0.0], [-np.inf, 1.0, 1.0], [LIM * v, 0.0, 0.0]])
    insert(0)
    ops.append(("carve", np.concatenate([rays, bad, _edge_points(v, 40, seed)]), c0, 1.0))
    insert(1)  # refills what went
    ops.append(("carve", rays, c0 + 0.3 * v, 1e-9))  # only t = 0: the origin's cell
    insert(2)
    ops.append(("carve", _centres([[4, 0, 0], [-4, 2, 0], [6, 6, 0], [3, -1, 2]], v), c0, 0.75))  # 0.75 * 4 = 3 exactly
    ops.append(("carve", _centres([[6, 0, 0], [0, -6, 6], [5, 5, 5]], v), c0, 0.5))
    insert(3)
    ops.append(("carve", _centres([[16384, 0, 0]], v), c0, 1.0))  # n = 16384: the whole line but its end
    insert(4)
    ops.append(("carve", _centres([[16385, 0, 0], [16385, 1, 0]], v), c0, 1.0))  # n = 16385: nothing
    ops.append(("carve", rays, np.array([LIM * v, 0.0, 0.0]), 1.0))  # the origin's key is out of range
    ops.append(("carve", rays, np.array([0.0, np.nan, 0.0]), 1.0))
    ops.append(("carve", _centres([[LIM - 1, 0, 0], [LIM - 1, 5, -5]], v), _centres([[LIM - 101, 0, 0]], v)[0], 1.0))
    ops.append(("carve", _centres([[-(LIM - 1), 0, 0]], v), _centres([[-(LIM - 50), 0, 0]], v)[0], 0.5))
    ops.append(("carve", _centres([[LIM - 1, LIM - 1, LIM - 1]], v), _centres([[LIM - 30, LIM - 30, LIM - 30]], v)[0],
                1.0))
    P = _edge_points(v, 200, seed=77 + seed) + rs.rand(200, 3) * 0.1 * v
    ops.append(("insert", P, 90, np.arange(200)))
    ops.append(("carve", P[:100], c0, 1.0))
    ops.append(("remove", c0, 8 * v))
    ops.append(("carve", P[100:], -c0, 0.9))
    return ops


def _apply(o, ops):
    for op in ops:
        if op[0] == "insert":
            o.insert(*op[1:])
        elif op[0] == "remove":
            o.remove_far(*op[1:])
        else:
            o.carve(*op[1:])


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_symbols_bound_and_abi_unchanged(built):
    L = _capi.lib()
    assert "madicp_map_carve" in _capi.SYMBOLS and L.madicp_map_carve.restype is not None
    assert L.madicp_abi_version() == 3


def test_bad_arguments_without_gpu(built):
    L = _capi.lib()
    fake = C.c_void_p(1)  # never dereferenced: the value checks come first
    assert L.madicp_map_carve(None, fake, None, 1.0) < 0
    assert b"null map" in L.madicp_last_error()
    assert L.madicp_map_carve(fake, None, None, 1.0) < 0
    assert b"null map or tree" in L.madicp_last_error()
    for r in (float("nan"), 0.0, -0.0, -1.0, 1.0000000000000002, 2.0, INF, -INF):
        assert L.madicp_map_carve(fake, fake, None, r) == -1, r  # MADICP_ERR_INVALID
        assert b"reach" in L.madicp_last_error()


@pytest.mark.parametrize("v,K", [(0.25, 1), (0.25, 3), (1.0, 2), (0.1, 32)])
def test_numpy_oracle_is_the_dict_loop(v, K):
    ops = _carve_ops(v, 0)
    o = CarveOracle(v, K)
    _apply(o, ops)
    xyz, sr = o.points()
    want_xyz, want_sr, dropped, live = dict_carve_oracle(ops, v, K)
    assert bits_equal(xyz, want_xyz) and (sr == want_sr).all() and o.dropped == dropped
    assert o.keys.size == live and want_xyz.shape[0] > 0 and o.removed > 0


def _one_ray(b, reach=1.0, origin=(0, 0, 0), v=0.25):
    """the cells a ray from cell `origin` to cell b carves in a block of filled voxels"""
    g = np.arange(-7, 8)
    block = _centres(np.stack(np.meshgrid(g, g, g, indexing="ij"), axis=-1).reshape(-1, 3), v)
    o = CarveOracle(v, 1)
    o.insert(block, 0, np.arange(block.shape[0]))
    before = set(o.keys.tolist())
    o.carve(_centres([b], v), _centres([origin], v)[0], reach)
    gone = before - set(o.keys.tolist())
    f = (1 << 21) - 1
    return sorted(((k & f) - LIM, ((k >> 21) & f) - LIM, (k >> 42) - LIM) for k in gone)


def test_the_line_at_its_edges():
    # floor_div(2 d t + n, 2 n) = floor(d t / n + 1/2): half-way ties go to the larger key, in both signs of d (the
    # true lines below pass y = +-0.5 at x = 1)
    assert _one_ray((2, 1, 0)) == [(0, 0, 0), (1, 1, 0)]
    assert _one_ray((2, -1, 0)) == [(0, 0, 0), (1, 0, 0)]
    assert _one_ray((-2, 1, 0)) == [(-1, 1, 0), (0, 0, 0)]
    assert _one_ray((6, -3, 3)) == [(0, 0, 0), (1, 0, 1), (2, -1, 1), (3, -1, 2), (4, -2, 2), (5, -2, 3)]
    assert _one_ray((-5, 0, 0)) == [(-t, 0, 0) for t in range(4, -1, -1)]
    assert _one_ray((-3, -3, 3)) == [(-2, -2, 2), (-1, -1, 1), (0, 0, 0)]
    assert _one_ray((0, 0, 0)) == []  # n = 0
    assert _one_ray((4, 0, 0), reach=0.75) == [(0, 0, 0), (1, 0, 0), (2, 0, 0)]  # 0.75 * 4 = 3: t < 3
    assert _one_ray((4, 0, 0), reach=0.7500000000000001) == [(t, 0, 0) for t in range(4)]
    assert _one_ray((6, 0, 0), reach=1e-300) == [(0, 0, 0)]
    assert _one_ray((5, 5, 0), origin=(-7, -7, 0)) == [(t, t, 0) for t in range(-7, 5)]
    # a ray of 16384 steps carves; one of 16385 does not
    v = 0.25
    line = _centres([[1, 0, 0], [16383, 0, 0], [16384, 0, 0], [16385, 0, 0]], v)
    for end, want in ((16384, 2), (16385, 0)):
        o = CarveOracle(v, 1)
        o.insert(line, 0, np.arange(4))
        o.carve(_centres([[end, 0, 0]], v), _centres([[0, 0, 0]], v)[0], 1.0)
        assert o.removed == want, end


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
    assert m.table()[2] == o.keys.size, what


def _nearest(xyz, q, r):
    """brute force: the least (d2, row) with d2 = ((x - qx)^2 + (y - qy)^2) + (z - qz)^2 <= r^2, else (-1, inf)"""
    row, best = np.full(q.shape[0], -1, np.int64), np.full(q.shape[0], INF)
    for i, p in enumerate(q):
        d = xyz - p
        d2 = (d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]
        ok = np.flatnonzero(d2 <= r * r)
        if ok.size:
            j = ok[np.lexsort((ok, d2[ok]))[0]]
            row[i], best[i] = j, d2[j]
    return row, best


@gpu
@pytest.mark.parametrize("v,K,reach", [(0.2, 1, 1.0), (0.5, 4, 0.75), (0.1, 32, 0.5), (0.3, 2, 1e-9)])
def test_engine_carve_is_the_oracle(drive, v, K, reach):
    reg, trees, clouds, poses = drive
    m = reg.voxel_map(v, K)  # reserve_points = 0: the map grows between carves
    o = CarveOracle(v, K)
    rs = np.random.RandomState(3)
    for s, (t, P, T) in enumerate(zip(trees, clouds, poses)):
        m.insert(t, T, scan=s)
        o.insert(_iso_apply(T, P), s, np.arange(P.shape[0]))
        _check(m, o, (s, "insert"))
        # a query before and after the carve: the second answers from the carved map (the row index was rebuilt)
        q = np.concatenate([o.points()[0][rs.choice(o.points()[0].shape[0], 150)], _iso_apply(T, P[:50])])
        q = q + rs.uniform(-0.5 * v, 0.5 * v, q.shape)
        got = m.nearest(q, v)
        want = _nearest(o.points()[0], q, v)
        assert (got[0] == want[0]).all() and bits_equal(got[1], want[1]), (s, "query before")
        removed = o.removed
        m.carve(t, T, reach)
        o.carve(_iso_apply(T, P), np.asarray(T)[:3, 3], reach)
        _check(m, o, (s, "carve"))
        got = m.nearest(q, v)
        want = _nearest(o.points()[0], q, v)
        assert (got[0] == want[0]).all() and bits_equal(got[1], want[1]), (s, "query after")
        if s > 0 and reach >= 0.5:  # (a tiny reach carves only the sensor's own voxel, which is mostly empty)
            assert o.removed > removed, s  # the carve took something
        if s % 2 == 1:
            m.remove_far(np.asarray(T)[:3, 3], 25.0)
            o.remove_far(np.asarray(T)[:3, 3], 25.0)
            _check(m, o, (s, "window"))
    # unposed: the rays start at the origin; the same carve again takes nothing more
    m.insert(trees[0], None, scan=20)
    o.insert(clouds[0], 20, np.arange(clouds[0].shape[0]))
    for _ in range(2):
        m.carve(trees[1], None, reach)
        o.carve(clouds[1], np.zeros(3), reach)
        _check(m, o, "unposed")
    # refills of carved voxels
    for s in (1, 2):
        m.insert(trees[s], poses[s - 1], scan=30 + s)
        o.insert(_iso_apply(poses[s - 1], clouds[s]), 30 + s, np.arange(clouds[s].shape[0]))
    _check(m, o, "refill")
    dx, ds = m.points(device=True)
    assert bits_equal(dx.cpu().numpy(), o.points()[0]) and (ds.cpu().numpy() == o.points()[1]).all()


@gpu
def test_engine_carve_rejects_bad_trees(built, drive):
    from mad_icp_b200 import Registrar
    reg, trees, clouds, poses = drive
    m = reg.voxel_map(0.2)
    m.insert(trees[0], None, scan=0)
    other = Registrar(device=0, max_keyframes=2)
    other.keep_cloud(True)
    t_other = other.build_tree(clouds[0])
    L = _capi.lib()
    assert L.madicp_map_carve(m._h, t_other._h, None, 1.0) == -1  # MADICP_ERR_INVALID
    assert b"another context" in L.madicp_last_error()
    reg.keep_cloud(False)
    try:
        bare = reg.build_tree(clouds[0])
    finally:
        reg.keep_cloud(True)
    assert L.madicp_map_carve(m._h, bare._h, None, 1.0) == -3  # MADICP_ERR_STATE
    assert b"kept no cloud" in L.madicp_last_error()
    o = CarveOracle(0.2, 1)
    o.insert(clouds[0], 0, np.arange(clouds[0].shape[0]))
    _check(m, o, "untouched")
    del t_other
    other.close()


@gpu
def test_long_rays_and_many_endpoints(drive):
    """rays of more than a warp's and a block's worth of steps (v = 0.05: up to 2000 steps), and one call with more
    endpoints than k_map_carve_mark's grid walks at once (1024 blocks of 8 warps of 32 rays)"""
    reg, trees, clouds, poses = drive
    v, K = 0.05, 2
    big = np.concatenate([_iso_apply(poses[s], clouds[s]) for s in range(6)] * 2)
    big = big + np.random.RandomState(0).uniform(-0.02, 0.02, big.shape)
    assert big.shape[0] > 1024 * 8 * 32
    t_big = reg.build_tree(big)
    m = reg.voxel_map(v, K)
    o = CarveOracle(v, K)
    for s in range(3):
        m.insert(trees[s], poses[s], scan=s)
        o.insert(_iso_apply(poses[s], clouds[s]), s, np.arange(clouds[s].shape[0]))
    m.carve(trees[3], poses[3], 1.0)
    o.carve(_iso_apply(poses[3], clouds[3]), poses[3][:3, 3], 1.0)
    _check(m, o, "long rays")
    kb, ok = _cells(_iso_apply(poses[3], clouds[3]), v)
    n = np.abs(kb[ok] - _cells(poses[3][:3, 3], v)[0]).max(axis=1)
    assert (n > 256).sum() > 1000 and n.max() <= MAX_RAY
    m.insert(t_big, None, scan=9)
    o.insert(big, 9, np.arange(big.shape[0]))
    before = o.removed
    T = synth.pose_xyyaw(10.0, 0.0, 0.0)  # (the endpoints are posed by T, as an insert would pose them)
    m.carve(t_big, T, 0.3)
    o.carve(_iso_apply(T, big), T[:3, 3], 0.3)
    assert o.removed > before
    _check(m, o, "many endpoints")


def _shell(n, radius, seed):
    """n points on a sphere of `radius` around the origin"""
    d = np.random.RandomState(seed).standard_normal((n, 3))
    return radius * d / np.linalg.norm(d, axis=1, keepdims=True)


@gpu
def test_churn_keeps_the_table_bounded(drive):
    """Every round inserts clutter on the cells of a shell's rays, then carves along them: the clutter goes, its
    tombstones pile up and the table is rebuilt from the live voxels, at a bounded size"""
    reg = drive[0]
    v, K, rounds, n_clutter = 0.5, 2, 120, 6000
    shell = _shell(3000, 20.0, 1)
    t_shell = reg.build_tree(shell)
    m = reg.voxel_map(v, K)
    o = CarveOracle(v, K)
    kb, _ = _cells(shell, v)
    nn = np.abs(kb).max(axis=1)
    created, peak_live, slots_seen = 0, 0, []
    for i in range(rounds):
        rs = np.random.RandomState(500 + i)
        j = rs.randint(0, shell.shape[0], n_clutter)  # a random inner step of a random ray
        t = (rs.rand(n_clutter) * 0.9 * nn[j]).astype(np.int64)
        k = (2 * kb[j] * t[:, None] + nn[j, None]) // (2 * nn[j, None])
        clutter = (k + rs.uniform(0.1, 0.9, k.shape)) * v
        before = set(o.keys.tolist())
        m.insert(reg.build_tree(clutter), None, scan=2 * i)
        o.insert(clutter, 2 * i, np.arange(n_clutter))
        m.insert(t_shell, None, scan=2 * i + 1)
        o.insert(shell, 2 * i + 1, np.arange(shell.shape[0]))
        created += len(set(o.keys.tolist()) - before)
        m.carve(t_shell, None, 1.0)
        o.carve(shell, np.zeros(3), 1.0)
        peak_live = max(peak_live, o.keys.size)
        if i % 20 == 19:
            slots, occupied, live = m.table()
            assert live == o.keys.size and 2 * occupied <= slots, i
            slots_seen.append(slots)
            _check(m, o, i)
    # many times more voxels went through the map than its table holds, and the table stayed within the policy's bound
    assert created >= 4 * max(slots_seen), (created, slots_seen)
    assert max(slots_seen) <= 8 * (peak_live + n_clutter), (slots_seen, peak_live)
    assert slots_seen[len(slots_seen) // 2:] == [slots_seen[-1]] * (len(slots_seen) - len(slots_seen) // 2)
    _check(m, o, "end")


# ----------------------------------------------------------------------------------------------------------- pipeline
@functools.lru_cache(maxsize=None)
def _seq(layout):
    return _sequence(24, layout)


@gpu
@pytest.mark.parametrize("reach", [0.5, 1.0])
@pytest.mark.parametrize("deskew", [False, True])
@pytest.mark.parametrize("case", ["kitti", "ouster"])
def test_pipeline_carve_is_the_oracle(built, case, deskew, reach):
    layout, gate, field, scale, mkw = CASES[case]
    seq = _seq(layout)
    p = _pipeline(deskew=deskew, keep=True, map_carve=reach, **mkw)
    ref = _pipeline(deskew=deskew, keep=True, map_carve=0.0, **mkw)
    o = CarveOracle(mkw["map_voxel_size"], mkw["map_points_per_voxel"])
    l0, r0 = p._kernelLaunches(), ref._kernelLaunches()
    for i, a in enumerate(seq):
        scan = p.currentID()
        p.computeRecords(0.1 * i, a, **gate)
        ref.computeRecords(0.1 * i, a, **gate)
        P = p.currentCloudArray(frame="map")
        o.insert(P, scan, p.currentCloudIndices())
        o.carve(P, p.currentPose()[:3, 3], reach)
        ref.currentCloudArray(frame="map")  # (the same reads on both: they launch too)
        ref.currentCloudIndices()
        assert bits_equal(p.currentPose(), ref.currentPose()), i  # registration is untouched
        assert p.keyframeID() == ref.keyframeID() and p.inliersRatio() == ref.inliersRatio(), i
        if i % 6 == 5:
            assert bits_equal(p.mapArray(), o.points()[0]) and (p.mapIndices() == o.points()[1]).all(), i
            ref.mapArray()
            ref.mapIndices()
    want_xyz, want_sr = o.points()
    assert p.mapSize() == want_xyz.shape[0] > 0 and p.mapDropped() == o.dropped and o.removed > 0
    assert bits_equal(p.mapArray(device=True).cpu().numpy(), want_xyz)
    assert (p.mapIndices(device=True).cpu().numpy() == want_sr).all()
    assert p.mapSize() < ref.mapSize()
    # launches: exactly the carve's per scan on top of the same pipeline without it, which made the same reads
    assert (p._kernelLaunches() - l0) - (ref._kernelLaunches() - r0) == CARVE_LAUNCHES * len(seq)


@gpu
def test_launches_window_and_rejections(built):
    seq = _seq("kitti")[:8]
    mkw = dict(map_voxel_size=0.3, map_points_per_voxel=3)
    plain = _pipeline(deskew=True, keep=False, **mkw)
    zero = _pipeline(deskew=True, keep=False, map_carve=0.0, **mkw)
    both = _pipeline(deskew=True, keep=True, map_carve=0.75, map_max_distance=10.0, **mkw)
    o = CarveOracle(0.3, 3)
    for i, a in enumerate(seq):
        for p in (plain, zero):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
        scan = both.currentID()
        both.computeRecords(0.1 * i, a, **KITTI_GATE)
        P = both.currentCloudArray(frame="map")
        o.insert(P, scan, both.currentCloudIndices())
        o.carve(P, both.currentPose()[:3, 3], 0.75)
        o.remove_far(both.currentPose()[:3, 3], 10.0)
    assert zero._kernelLaunches() == plain._kernelLaunches()
    assert bits_equal(zero.mapArray(), plain.mapArray())
    assert bits_equal(both.mapArray(), o.points()[0]) and (both.mapIndices() == o.points()[1]).all()
    for bad in (dict(map_voxel_size=0.2, map_carve=-0.1), dict(map_voxel_size=0.2, map_carve=float("nan")),
                dict(map_voxel_size=0.2, map_carve=1.0000000000000002), dict(map_voxel_size=0.2, map_carve=INF),
                dict(map_carve=0.5)):
        with raises_madicp("map_carve"):
            _pipeline(**bad)


# ----------------------------------------------------------------------------------------------------------- behaviour
# A car parked beside the lane, present in the first scans of a drive and gone afterwards.  The lane (y around 1) is kept
# free by StreetScene; the car stands at x 8 .. 12.2, y 3.0 .. 4.8, 1.5 m high, where this scene has no other box, 2-4 m
# from a sensor 1.73 m above the ground that drives from x = 0 to 23 along the lane.  After it leaves, the sensor's
# downward rays to the ground beyond the car (y > 4.8) and its rays to the canyon wall at y = 12 cross the car's volume
# from many positions, so every voxel of its surface that does not also hold later ground points lies on later rays.
# The car is seen only on its faces, so the region checked is its box grown by 5 cm (five times the range noise), not
# shrunk: a box shrunk by a voxel per face holds no row in either run.  The lowest voxel layer is left out of the first
# check, since the ground under the car is seen, and mapped, once the car has gone.
CAR = (8.0, 12.2, 3.0, 4.8, 0.0, 1.5)
CAR_SCANS, DRIVE_SCANS = 6, 30


@functools.lru_cache(maxsize=None)
def _car_drive():
    scene = synth.StreetScene(seed=5, x_min=-45.0, x_max=90.0)
    gone = synth.StreetScene(seed=5, x_min=-45.0, x_max=90.0)
    b = scene.boxes
    assert not ((b[:, 0] < CAR[1]) & (b[:, 1] > CAR[0]) & (b[:, 2] < CAR[3]) & (b[:, 3] > CAR[2])).any()
    scene.boxes = np.vstack([b, np.array(CAR)])
    out = []
    for i in range(DRIVE_SCANS):
        base = synth.pose_xyyaw(0.8 * i, 1.0, 0.0)
        p = synth.lidar_scan(scene if i < CAR_SCANS else gone, base, beams=32, azimuths=1024, seed=300 + i)
        a = np.zeros((p.shape[0], 4), np.float32)
        a[:, :3] = p
        out.append(a)
    return out


def _in_car(xyz, v, above_ground=True):
    """rows inside the car's box grown by 5 cm, optionally above its lowest voxel, in the map frame (the first scan's
    sensor frame: the world moved by -(0, 1, 1.73))"""
    lo = np.array(CAR[0::2]) - np.array([0.0, 1.0, 1.73]) - 0.05
    hi = np.array(CAR[1::2]) - np.array([0.0, 1.0, 1.73]) + 0.05
    if above_ground:
        lo[2] += v + 0.05
    return ((xyz > lo) & (xyz < hi)).all(axis=1)


@gpu
def test_a_car_that_left_leaves_no_trace(built):
    v = 0.2
    runs = {}
    for reach in (0.0, 1.0):
        p = _pipeline(deskew=False, keep=True, map_voxel_size=v, map_points_per_voxel=4, map_carve=reach)
        for i, a in enumerate(_car_drive()):
            p.computeRecords(0.1 * i, a, **KITTI_GATE)
        runs[reach] = (p.mapArray(), p.mapIndices(), p.trajectory())
    off, on = runs[0.0], runs[1.0]
    assert bits_equal(np.array(off[2]), np.array(on[2]))  # the same poses
    car_off = _in_car(off[0], v)
    assert car_off.sum() > 1000 and (off[1][car_off, 0] < CAR_SCANS).all()  # the car's points stay without carving
    assert not _in_car(on[0], v).any()  # and go with it
    assert not (on[1][_in_car(on[0], v, above_ground=False), 0] < CAR_SCANS).any()  # not one row the car scans left
