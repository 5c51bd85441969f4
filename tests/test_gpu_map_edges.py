"""The voxel map's keys, window and queries on the device at their edges, and at the sizes where their one-CTA passes
loop, bit for bit against the oracles of test_gpu_voxel_map, test_gpu_map_window and test_gpu_map_query (`-m gpu`).

  A  edge keys: fields at +-(2^20 - 1) on every axis, -0.0, exact voxel boundaries, quotients that round up onto a key,
     NaN and inf, through the insert (k_map_claim), the removal (k_map_evict unpacks the keys) and the query (its box
     clamped at +-(2^20 - 1) next to real rows), with ties of the removal rule;
  B  (query, row) pairs a few ulps around cell boundaries whose row sits on the first or last key of the query's box
     (the -1 / +1 of first() / last() in k_mapq_nearest), at exactly r and one ulp beyond;
  C  a map of more than 1 047 552 rows (k_map_evict_sums loops) in a table of at least 2^21 slots (k_mapq_sums loops),
     removals whose first removed row lies past the first 1024 tiles, at row 0, in the last tile only, of everything and
     of nothing, one enqueued behind an insert still waiting on the stream, queries on the tombstone-heavy table, and
     a tombstone-dropping rebuild at millions of slots;
  D  a long windowed drive with queries, whose table settles;
  E  two maps on one Registrar, and inserts across the reset of the round tags.

Every case asserts, from the oracle or from `table()`, that its input reaches what it is there for."""
import math
from fractions import Fraction

import numpy as np
import pytest

from mad_icp_b200 import Registrar, _capi, synth
from test_gpu_map_query import _check_all, _same, nearest_loop, nearest_oracle
from test_gpu_map_query import _edge_case
from test_gpu_map_window import WindowOracle, _far, _ops
from test_gpu_voxel_map import LIM, MapOracle, _edge_points, _iso_apply
from util import bits_equal

gpu = pytest.mark.gpu
INF = float("inf")
V_EDGE = [0.25, 0.1, 0.3, 1 / 3]
V_BOX = [0.1, 0.3, 1 / 3, 0.7]
EVICT_ONE_PASS = 1023 * 1024  # k_map_evict_sums scans n_tiles + 1 row-tile totals: one pass up to this many rows
QUERY_TWO_PASS = 1 << 21      # k_mapq_sums scans slots / 1024 totals: a second pass from this many slots on
FIRST_TILES = 1 << 20         # rows of the first 1024 tiles


# ----------------------------------------------------------------------------------------------------------- helpers
def _fields(xyz, v):
    """the key fields of each row as the map computes them: floor(RN(x / v)) per axis"""
    with np.errstate(invalid="ignore", over="ignore"):
        return np.floor(np.asarray(xyz, np.float64) / v)


def _dyadic(v):
    return np.frexp(v)[0] == 0.5  # a power of two: x / v is exact


def _unpose(T, P):
    """R^T (p - t): a tree input whose points the pose T takes to about P"""
    X = np.asarray(T, np.float64)[:3]
    with np.errstate(invalid="ignore"):
        return (P - X[:, 3]) @ X[:, :3]


def _same_map(m, o, what):
    """rows, (scan, record), size, drops and the table's live voxels, bit for bit"""
    want_xyz, want_sr = o.points()
    assert m.size() == want_xyz.shape[0], what
    assert m.dropped() == o.dropped, what
    xyz, sr = m.points()
    assert bits_equal(xyz, want_xyz) and (sr == want_sr).all(), what
    slots, occupied, live = m.table()
    assert live == o.keys.size and live <= occupied and 2 * occupied <= slots, (what, slots, occupied, live)
    return slots, occupied, live


def _round_up(v, seed, n=64):
    """coordinates x < k v (as exact rationals) whose quotient RN(x / v) rounds up onto k, so that their key is k and not
    k - 1: stepping ulps down from RN(k v) for keys across the whole range (there are none for a power-of-two v)"""
    k = np.random.RandomState(seed).randint(-(LIM - 1), LIM, size=4000).astype(np.float64)
    x, out = k * v, []
    for _ in range(6):
        for i in np.flatnonzero(np.floor(x / v) == k):
            if Fraction(float(x[i])) < int(k[i]) * Fraction(v):
                out.append(float(x[i]))
        x = np.nextafter(x, -INF)
    return np.array(out[:n])


def _rounds_up(xyz, v):
    """rows with a finite coordinate x < key(x) v exactly"""
    f = _fields(xyz, v)
    hit = np.zeros(xyz.shape[0], bool)
    for i, a in zip(*np.nonzero(np.isfinite(xyz) & (xyz != 0.0))):
        hit[i] |= Fraction(float(xyz[i, a])) < int(f[i, a]) * Fraction(v)
    return hit


def _edge_cloud(v, seed):
    """_edge_points, a row at the centre, the low boundary and the top of a voxel whose field is +-(2^20 - 1) on each
    axis, and the round-up coordinates of _round_up on random axes"""
    rs = np.random.RandomState(seed)
    ext = []
    for a in range(3):
        for s in (-1, 1):
            for frac in (0.5, 0.0, 0.999):
                p = (rs.randint(-8, 8, size=3) + 0.5) * v
                p[a] = (s * (LIM - 1) + frac) * v
                ext.append(p)
    up = _round_up(v, seed)
    U = (rs.randint(-8, 8, size=(up.size, 3)) + 0.5) * v
    U[np.arange(up.size), rs.randint(0, 3, size=up.size)] = up
    return np.concatenate([_edge_points(v, 400, seed), np.array(ext), U])


def _ties(v, origin, D):
    """centres of the voxels around the origin whose centre lies at exactly D by the removal's arithmetic (ties: they
    stay)"""
    if not math.isfinite(D):
        return np.empty((0, 3))
    g = np.arange(-13, 14)
    k = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + np.floor(np.asarray(origin) / v)
    k = k[(np.abs(k) < LIM - 1).all(axis=1)]
    d = (k + 0.5) * v - np.asarray(origin, np.float64)
    return (k[((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) == np.float64(D) * np.float64(D)] + 0.5) * v


def _key_fields(keys):
    f = (1 << 21) - 1
    return np.column_stack([keys & f, (keys >> 21) & f, keys >> 42]) - LIM


@pytest.fixture(scope="module")
def reg(built):
    """a Registrar that keeps the clouds of the trees it builds"""
    r = Registrar(device=0, max_keyframes=2)
    r.keep_cloud(True)
    return r


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_edge_inputs_reach_their_edges():
    """the fixtures of A: fields at both extremes on every axis, round-up coordinates for every v that is not a power of
    two, -0.0, and ties of the removal rule in the _ops sequence"""
    for v in V_EDGE:
        P = _edge_cloud(v, seed=1)
        o = MapOracle(v, 3)
        o.insert(P, 0, np.arange(P.shape[0]))
        xyz, _ = o.points()
        f = _fields(xyz, v)
        for a in range(3):
            assert (f[:, a] == LIM - 1).any() and (f[:, a] == -(LIM - 1)).any(), (v, a)
        assert ((xyz == 0.0) & np.signbit(xyz)).any()
        assert _rounds_up(xyz, v).any() != _dyadic(v), v
        assert sum(_ties(v, *op[1:]).shape[0] for op in _ops(v, 0) if op[0] == "remove") > 0, v


def test_set_rounds_without_gpu(built):
    L = _capi.lib()
    assert L.madicp_debug_map_set_rounds(None, 0) < 0
    assert b"null map" in L.madicp_last_error()


# ----------------------------------------------------------------------------------------------------------- A
@gpu
@pytest.mark.parametrize("v", V_EDGE)
def test_edge_keys_insert(reg, v):
    """unposed and posed inserts of edge clouds: every key field at both extremes, -0.0 kept as -0.0, round-up keys"""
    P = _edge_cloud(v, seed=1)
    T = synth.pose_xyyaw(0.7, -1.3, 0.4, z=0.2)
    Pin = _unpose(T, P)
    posed = _iso_apply(T, Pin)
    tp, tq = reg.build_tree(P), reg.build_tree(Pin)
    assert bits_equal(tp.cloud()[0], P)  # NaN and inf reach the map
    for K in (1, 3):
        m, o = reg.voxel_map(v, K), MapOracle(v, K)
        for s, (t, X, pts) in enumerate([(tp, None, P), (tq, T, posed), (tp, None, P)]):
            m.insert(t, X, scan=s)
            o.insert(pts, s, np.arange(pts.shape[0]))
            _same_map(m, o, (v, K, s))
        xyz, sr = o.points()
        # the rows of the first insert and the posed points of the second (which a wrong key would add as rows)
        for f in (_fields(xyz[sr[:, 0] == 0], v), _fields(posed, v)):
            for a in range(3):
                for sign in (-1, 1):
                    assert (f[:, a] == sign * (LIM - 1)).any(), (K, a, sign)
        assert ((xyz == 0.0) & np.signbit(xyz))[sr[:, 0] == 0].any()  # (bits_equal tells -0.0 from 0.0)
        assert o.dropped > 0 and (K == 1 or (o.counts > 1).any())
        assert _rounds_up(xyz[sr[:, 0] == 0], v).any() != _dyadic(v)
        m.free()


@gpu
@pytest.mark.parametrize("v", V_EDGE)
def test_edge_keys_window(reg, v):
    """the whole _ops sequence, with the voxels that tie each removal's D added, against WindowOracle; the table after
    every removal; removed keys with every field at both extremes, and ties that stay"""
    for K in (1, 3):
        m, o = reg.voxel_map(v, K), WindowOracle(v, K)
        ops = _ops(v, seed=K)
        gone, ties = [], 0
        for i, op in enumerate(ops):
            if op[0] == "insert":
                P = op[1]
                if i + 1 < len(ops):
                    P = np.concatenate([P, _ties(v, *ops[i + 1][1:])])
                m.insert(reg.build_tree(P), None, scan=op[2])
                o.insert(P, op[2], np.arange(P.shape[0]))
                continue
            origin, D = op[1:]
            before = o.keys
            if math.isfinite(D):
                k = _key_fields(before)
                d = (k + 0.5) * v - np.asarray(origin, np.float64)
                ties += int((((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2]) == D * D).sum())
            m.remove_far(origin, D)
            o.remove_far(origin, D)
            gone.append(np.setdiff1d(before, o.keys))
            _same_map(m, o, (v, K, i))
        f = _key_fields(np.concatenate(gone))
        for a in range(3):
            assert (f[:, a] == LIM - 1).any() and (f[:, a] == -(LIM - 1)).any(), (K, a)
        assert ties > 0 and o.removed > 0
        m.free()


@gpu
@pytest.mark.parametrize("v", V_EDGE)
def test_edge_keys_query(reg, v):
    """_edge_case's map and queries, and queries within r of the rows at the extreme keys, whose box the clamp cuts, at
    r in {0, v/2, v, 4v} in host and float32 / float64 strided device form, with and without scan_below"""
    xyz, sr, Q = _edge_case(v)
    m, o = reg.voxel_map(v, 3), MapOracle(v, 3)
    for s in np.unique(sr[:, 0]):  # (the scans in insertion order: each voxel holds <= 3 rows, so every row stays)
        rows = xyz[sr[:, 0] == s]
        m.insert(reg.build_tree(rows), None, scan=int(s))
        o.insert(rows, int(s), np.arange(rows.shape[0]))
    assert bits_equal(o.points()[0], xyz) and (o.points()[1][:, 0] == sr[:, 0]).all()
    _same_map(m, o, v)
    f = _fields(xyz, v)
    rs = np.random.RandomState(5)
    near = []
    for i, a in zip(*np.nonzero(np.abs(f) == LIM - 1)):
        for step in (0.0, 0.4, 1.2, 2.5, 3.9):
            q = xyz[i] + rs.uniform(-0.2, 0.2, 3) * v
            q[a] = xyz[i, a] + np.sign(f[i, a]) * step * v  # outwards, up to past the key limit
            near.append(q)
    Q = np.concatenate([Q, np.array(near)])
    clamped = set()
    for r in (v, 4 * v):
        row, _ = nearest_oracle(xyz, sr, Q, r)
        hit = np.flatnonzero(row >= 0)
        hf, qa = f[row[hit]], Q[hit]
        last, first = np.floor((qa + r) / v) + 1, np.floor((qa - r) / v) - 1
        for a in range(3):
            if ((hf[:, a] == LIM - 1) & (last[:, a] > LIM - 1)).any():
                clamped.add((a, 1))
            if ((hf[:, a] == -(LIM - 1)) & (first[:, a] < -(LIM - 1))).any():
                clamped.add((a, -1))
    assert clamped == {(a, s) for a in range(3) for s in (-1, 1)}, clamped
    for below in (None, 8):
        _check_all(m, o, Q, v, ("edge", v), scan_below=below)
    m.free()


# ----------------------------------------------------------------------------------------------------------- B
def _step(x, n):
    for _ in range(abs(n)):
        x = np.nextafter(x, INF if n > 0 else -INF)
    return x


def _box_pairs(v, U=6):
    """(row coordinate, query coordinate, m, kind) along one axis for r = m v, m = 1..4: the row RN(k v) stepped by up to
    U ulps for keys k in [-64, 64], the query RN(row -+ r) stepped by up to U ulps.  Kinds: 0 the row's key is the first
    key of the query's box, 1 the last, 2 the row at exactly r (d2 == r2), 3 one ulp beyond such a row.  Kinds 0-2 are
    kept when d2 <= r2; at most 24 pairs of kind 2 per m.  Also returns the qualifying pairs that the cell bound would
    prune without its 2^-20 margin."""
    k = np.arange(-64, 65, dtype=np.float64)
    rs = np.random.RandomState(int(v * 1000))
    out, margin = [], 0
    for m in (1, 2, 3, 4):
        r = m * v
        exact = []
        for i in range(-U, U + 1):
            x = _step(k * v, i)
            kx = np.floor(x / v)
            for j in range(-U, U + 1):
                for kind, q in ((0, _step(x + r, j)), (1, _step(x - r, j))):
                    dx = x - q
                    ok = dx * dx <= r * r
                    box = np.floor((q - r) / v) - 1 if kind == 0 else np.floor((q + r) / v) + 1
                    out += [(x[s], q[s], m, kind) for s in np.flatnonzero(ok & (kx == box))]
                    exact += [(x[s], q[s]) for s in np.flatnonzero(ok & (dx * dx == r * r))]
                    g = np.maximum(np.abs(kx - np.floor(q / v)) - 1.0, 0.0)
                    margin += int((ok & (g * g > (r / v) * (r / v))).sum())
        for s in rs.choice(len(exact), min(24, len(exact)), replace=False):
            x, q = exact[s]
            out += [(x, q, m, 2), (float(_step(np.float64(x), 1 if x > q else -1)), q, m, 3)]
    return out, margin


def _box_map(v):
    """rows and queries of _box_pairs in 3-d: pair p along axis p % 3, in a lane of its own (the other two coordinates,
    shared by row and query, 11 v from any other lane), each checked alone by the loop oracle"""
    pairs, margin = _box_pairs(v)
    rows, qs, meta = [], [], []
    for p, (x, q, m, kind) in enumerate(pairs):
        a = p % 3
        lane = (np.array([p % 512 - 256, p // 512 - 8]) * 11 + 0.5) * v
        row, qq = np.insert(lane, a, x), np.insert(lane, a, q)
        got, _ = nearest_loop(row[None], np.zeros((1, 2), np.int64), qq[None], m * v)
        if got[0] == 0 or kind == 3:
            rows.append(row)
            qs.append(qq)
            meta.append((m, kind, got[0] == 0))
    return np.array(rows), np.array(qs), np.array(meta, np.int64), margin


def test_box_pairs_reach_the_box_edges():
    """Rows on the first key of the box at every r, on the last key at some r, at exactly r, and one ulp beyond r
    rejected.  At v = 0.7, r = 3 v the search also finds 2 qualifying pairs whose cell the pruning bound would skip
    without its 2^-20 margin (r / v rounds to 2.9999999999999996 there); that is recorded, not required."""
    for v in V_BOX:
        rows, qs, meta, margin = _box_map(v)
        for m in (1, 2, 3, 4):
            sel = meta[:, 0] == m
            assert ((meta[:, 1] == 0) & sel).any() and ((meta[:, 1] == 2) & sel).any(), (v, m)
            assert ((meta[:, 1] == 3) & sel & (meta[:, 2] == 0)).any(), (v, m)
        assert (meta[:, 1] == 1).any(), v
        print(f"v = {v}: {int((meta[:, 1] == 0).sum())} first-key and {int((meta[:, 1] == 1).sum())} last-key pairs, "
              f"{margin} that need the bound's margin")


@gpu
@pytest.mark.parametrize("v", V_BOX)
def test_box_edges_on_the_device(reg, v):
    import torch
    rows, qs, meta, _ = _box_map(v)
    m, o = reg.voxel_map(v, 2), MapOracle(v, 2)
    m.insert(reg.build_tree(rows), None, scan=0)
    o.insert(rows, 0, np.arange(rows.shape[0]))
    _same_map(m, o, v)
    xyz, sr = o.points()
    own, last = np.arange(qs.shape[0]), 0
    for mult in (1, 2, 3, 4):
        r = mult * v
        want = nearest_oracle(xyz, sr, qs, r)
        _same(m.nearest(qs, r), want, (v, r, "host"))
        _same(m.nearest(torch.from_numpy(qs).cuda(), r), want, (v, r, "device"))
        mine = (meta[:, 0] == mult) & (want[0] == own)  # the answer is the pair's own row
        assert (mine & (meta[:, 1] == 0)).any() and (mine & (meta[:, 1] == 2)).any(), (v, r)
        assert ((meta[:, 0] == mult) & (meta[:, 1] == 3) & (want[0] == -1)).any(), (v, r)
        last += int((mine & (meta[:, 1] == 1)).sum())
    assert last > 0
    m.free()


# ----------------------------------------------------------------------------------------------------------- C
N_BIG = (1 << 20) + (1 << 16)  # one tree, inserted under several translations


@gpu
def test_passes_that_loop(reg):
    import torch
    v, K = 0.1, 1
    base = np.random.RandomState(17).uniform(0.0, 1.0, (N_BIG, 3)) * np.array([200.0, 200.0, 20.0])
    tree = reg.build_tree(base)
    m, o = reg.voxel_map(v, K), WindowOracle(v, K)
    centre = np.array([100.0, 100.0, 10.0])

    def insert(t, pts, x, scan):
        T = np.eye(4)
        T[0, 3] = x
        m.insert(t, T, scan=scan)
        o.insert(_iso_apply(T, pts), scan, np.arange(pts.shape[0]))

    def remove(origin, D):
        """the removal on both; returns the rows it took (indices before it)"""
        xyz, _ = o.points()
        gone = np.flatnonzero(_far(_fields(xyz, v), v, origin, D))
        m.remove_far(origin, D)
        o.remove_far(origin, D)
        return gone

    def queries(what):
        rs = np.random.RandomState(len(what))
        xyz, sr = o.points()
        Q = xyz[rs.choice(xyz.shape[0], 1 << 17)]
        Q[: 1 << 16] += rs.uniform(-0.5 * v, 0.5 * v, (1 << 16, 3))  # (within v of their row)
        Q[1 << 16:] += rs.uniform(-4 * v, 4 * v, (1 << 16, 3))
        below = int(np.median(sr[:, 0])) + 1
        for r, sb in ((v, below), (4 * v, below), (v, None)):
            want = nearest_oracle(xyz, sr, Q, r, sb)
            _same(m.nearest(Q, r, sb), want, (what, r, sb, "host"))
            _same(m.nearest(torch.from_numpy(Q).cuda(), r, sb), want, (what, r, sb, "device"))
            assert (want[0] >= 0).mean() > 0.2 and (sb is None or (want[0] >= 0).sum() < (want[0] >= 0).size)

    insert(tree, base, 0.0, 0)
    rows0 = o.points()[0].shape[0]
    insert(tree, base, 1000.0, 1)
    slots, _, _ = _same_map(m, o, "two inserts")
    assert rows0 > FIRST_TILES and m.size() > EVICT_ONE_PASS and slots >= QUERY_TWO_PASS

    # nothing goes: 5 launches, the same rows
    before = m.points()
    l0 = reg.kernel_launches
    assert remove(centre, 1.0e4).size == 0
    assert reg.kernel_launches - l0 == 5
    after = m.points()
    assert bits_equal(after[0], before[0]) and (after[1] == before[1]).all()
    _same_map(m, o, "nothing")

    # part of the second box: the first removed row lies past the first 1024 tiles, and rows after it move
    gone = remove(centre, 1050.0)
    assert gone.size and gone[0] > FIRST_TILES and gone[-1] - gone[0] + 1 > gone.size, (gone[:1], gone.size)
    _same_map(m, o, "tail")
    slots, occupied, live = m.table()
    assert occupied - live > 100_000 and slots >= QUERY_TWO_PASS  # a tombstone-heavy table
    queries("tail")

    # row 0's voxel goes (and every voxel farther than it): the compaction starts at row 0
    xyz, _ = o.points()
    d = (_fields(xyz[:1], v) + 0.5) * v - centre
    D = math.sqrt((d[0, 0] * d[0, 0] + d[0, 1] * d[0, 1]) + d[0, 2] * d[0, 2]) * (1 - 1e-12)
    gone = remove(centre, D)
    assert gone.size and gone[0] == 0 and gone.size < xyz.shape[0]
    _same_map(m, o, "row 0")

    # an insert held behind work on the map's stream and a removal enqueued after it before the insert ran: the removal
    # takes only rows of the last tile.  The table and the rows have room, so neither call waits for the stream.
    M = o.points()[0].shape[0]
    n_s = min(37, 1024 - M % 1024)
    small = np.random.RandomState(3).uniform(0.0, 1.0, (n_s, 3)) + np.array([3000.0, 0.0, 0.0])
    t_small = reg.build_tree(small)
    slots, occupied, live = m.table()
    assert 2 * (occupied + n_s) <= slots and M + n_s <= 2 * N_BIG
    stream = torch.cuda.ExternalStream(reg.stream)
    with torch.cuda.stream(stream):
        torch.cuda._sleep(2_000_000_000)  # (about a second)
        held = torch.cuda.Event()
        held.record(stream)
    insert(t_small, small, 0.0, 2)
    added = o.points()[0].shape[0] - M
    gone = remove(centre, 500.0)
    assert not held.query()  # both calls returned while the stream still slept
    assert 0 < gone.size == added and gone[0] >= 1024 * ((M + added - 1) // 1024), (gone, M)
    _same_map(m, o, "last tile")

    # churn: boxes farther and farther along x, each removal taking the box before, until an insert rebuilds the table
    # from its live voxels (fewer occupied slots after it)
    occupied = m.table()[1]
    for j in range(8):
        x = 2000.0 * (j + 1)
        insert(tree, base, x, 10 + j)
        slots, occ, live = m.table()
        if occ < occupied:
            break
        remove(centre + [x, 0.0, 0.0], 400.0)
        occupied = m.table()[1]
    else:
        pytest.fail("no rebuild")
    assert slots >= 1 << 22 and occ == live, (slots, occ, live)
    _same_map(m, o, "rebuild")
    queries("rebuild")
    gone = remove(centre + [x + 150.0, 0.0, 0.0], 120.0)
    assert gone.size
    _same_map(m, o, "after the rebuild")
    queries("after the rebuild")

    # everything goes; then the map fills again
    gone = remove([1.0e5, 0.0, 0.0], 10.0)
    assert gone.size and m.size() == 0 and m.table()[2] == 0
    _same_map(m, o, "everything")
    insert(t_small, small, 0.0, 99)
    _same_map(m, o, "refill")
    m.free()


# ----------------------------------------------------------------------------------------------------------- D
@gpu
def test_long_windowed_drive(reg):
    """180 posed inserts of three 64 x 2048 scans along a path, remove_far(D = 50) after each, a query with the next
    scan's points at scan_below = the current scan every 10 scans: the oracles, and a table whose size settles"""
    import torch
    scene = synth.StreetScene(seed=13, x_min=-70.0, x_max=70.0)
    scans = [synth.lidar_scan(scene, synth.pose_xyyaw(0.0, 0.5 * k, 0.02 * k), beams=64, azimuths=2048, seed=500 + k)
             for k in range(3)]
    trees = [reg.build_tree(P) for P in scans]
    v, K, D, n = 0.3, 2, 50.0, 180
    poses = [synth.pose_xyyaw(3.0 * i, 4.0 * math.sin(0.02 * i), 0.3 * math.sin(0.01 * i), z=0.1 * math.sin(0.05 * i))
             for i in range(n + 1)]
    m, o = reg.voxel_map(v, K), WindowOracle(v, K)
    slots_seen, hits, rebuilds, occupied = [], 0, 0, 0
    for i in range(n):
        m.insert(trees[i % 3], poses[i], scan=i)
        o.insert(_iso_apply(poses[i], scans[i % 3]), i, np.arange(scans[i % 3].shape[0]))
        origin = np.asarray(poses[i])[:3, 3]
        m.remove_far(origin, D)
        o.remove_far(origin, D)
        if i % 10 == 9:
            Q = _iso_apply(poses[i + 1], scans[(i + 1) % 3])
            xyz, sr = o.points()
            want = nearest_oracle(xyz, sr, Q, v, scan_below=i)
            _same(m.nearest(torch.from_numpy(Q).cuda() if i % 20 == 19 else Q, v, scan_below=i), want, i)
            hits += int((want[0] >= 0).sum())
            slots, occ, live = m.table()
            assert live == o.keys.size, i
            rebuilds += occ < occupied
            occupied = occ
            slots_seen.append(slots)
        if i % 30 == 29:
            _same_map(m, o, i)
    assert o.removed > 0 and hits > 0
    # more voxels went through the map than its table has slots, the table was rebuilt from its live voxels again and
    # again, and its size settled
    assert o.removed + o.keys.size > max(slots_seen) and rebuilds >= 2, (o.removed, o.keys.size, slots_seen, rebuilds)
    half = len(slots_seen) // 2
    assert slots_seen[half:] == [slots_seen[-1]] * (len(slots_seen) - half), slots_seen
    _same_map(m, o, "end")
    m.free()


# ----------------------------------------------------------------------------------------------------------- E
@gpu
def test_two_maps_on_one_registrar(reg):
    """inserts, removals and device queries of two maps interleaved without reading either map: each is its own
    oracle's (the counters' mirror, the operation count and the row index are per map)"""
    import torch
    scene = synth.StreetScene(seed=9, x_min=-45.0, x_max=90.0)
    clouds = [synth.lidar_scan(scene, synth.pose_xyyaw(0.0, 0.5, 0.0), beams=32, azimuths=1024, seed=60 + i)
              for i in range(6)]
    trees = [reg.build_tree(P) for P in clouds]
    poses = [synth.pose_xyyaw(6.0 * i, 0.3 * math.sin(i), 0.1 * i) for i in range(6)]
    a, oa = reg.voxel_map(0.2, 1, 1 << 20), WindowOracle(0.2, 1)
    b, ob = reg.voxel_map(0.5, 4, 1 << 20), WindowOracle(0.5, 4)
    pending = []
    for s in range(6):
        T, U = poses[s], poses[(s + 3) % 6]
        a.insert(trees[s], T, scan=s)
        oa.insert(_iso_apply(T, clouds[s]), s, np.arange(clouds[s].shape[0]))
        b.insert(trees[5 - s], U, scan=10 + s)
        ob.insert(_iso_apply(U, clouds[5 - s]), 10 + s, np.arange(clouds[5 - s].shape[0]))
        Q = _iso_apply(poses[(s + 1) % 6], clouds[(s + 2) % 6])[::7]
        for mp, o, r in ((a, oa, 0.2), (b, ob, 1.0)):
            pending.append((mp.nearest(torch.from_numpy(Q).cuda(), r), nearest_oracle(*o.points(), Q, r), (s, r)))
        a.remove_far(np.asarray(T)[:3, 3], 12.0)
        oa.remove_far(np.asarray(T)[:3, 3], 12.0)
        if s % 2:
            b.remove_far(np.asarray(U)[:3, 3], 15.0)
            ob.remove_far(np.asarray(U)[:3, 3], 15.0)
    torch.cuda.synchronize()
    for got, want, what in pending:
        _same(got, want, what)
    assert sum(int((w[0] >= 0).sum()) for _, w, _ in pending) > 0 and oa.removed > 0 and ob.removed > 0
    _same_map(a, oa, "a")
    _same_map(b, ob, "b")
    a.free()
    b.free()


@gpu
@pytest.mark.parametrize("K", [1, 3, 32])
def test_round_tags_run_out(reg, K):
    """inserts across the reset of the round words that madicp_map_insert makes when fewer than K tags are left (the
    count moved forward by madicp_debug_map_set_rounds), with voxels part full on both sides of it"""
    L = _capi.lib()
    v = 0.25
    rs = np.random.RandomState(K)
    # a core of 64 voxels that fills at every K, and a halo of 4096 that fills slowly
    clouds = [np.concatenate([rs.uniform(0.0, 1.0, (1500, 3)), rs.uniform(0.0, 4.0, (1500, 3))]) for _ in range(6)]
    trees = [reg.build_tree(P) for P in clouds]
    m, o = reg.voxel_map(v, K, 1 << 16), MapOracle(v, K)  # (room for every insert: a table growth resets the count)
    m.insert(trees[0], None, scan=0)
    o.insert(clouds[0], 0, np.arange(3000))
    jump = 0xFFFFFF00 - 3 * K + 1  # the third insert from here finds fewer than K tags left
    assert L.madicp_debug_map_set_rounds(m._h, jump) == K
    assert L.madicp_debug_map_set_rounds(m._h, jump - 1) < 0 and b"rounds must lie" in L.madicp_last_error()
    assert L.madicp_debug_map_set_rounds(m._h, 0xFFFFFF01) < 0
    want = [jump + K, jump + 2 * K, K, 2 * K, 3 * K]
    for s in range(1, 6):
        if s == 3:  # the reset: voxels with room left, which this insert adds to
            part = o.keys[(o.counts > 0) & (o.counts < K)]
            counts = dict(zip(o.keys.tolist(), o.counts.tolist()))
        m.insert(trees[s], None, scan=s)
        o.insert(clouds[s], s, np.arange(3000))
        assert L.madicp_debug_map_set_rounds(m._h, -1) == want[s - 1], s
        _same_map(m, o, (K, s))
    if K > 1:
        grown = [k for k in part.tolist() if o.counts[np.searchsorted(o.keys, k)] > counts[k]]
        assert part.size and grown
    assert (o.counts == K).any()
    m.free()
