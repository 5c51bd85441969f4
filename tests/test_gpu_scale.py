"""The device tree build, the scan ingest and the voxel map at the sizes of a look-ahead forest and of the per-cloud limit,
bit for bit against the host builds (`-m gpu`).

Many kernels of the device build use a fixed grid, or one CTA that loops in passes; their second iteration runs only
above a size threshold (the launch configurations of build_forest in gpu_tree.cu, tile_scan.cuh, voxel_map.cu):

  k_sums_big grid-stride (1776 CTAs)               a level with a node of >= 512 points at index >= 1776
  k_decide_mark / k_decide_apply (64 x 1024)       a level of > 65 536 nodes
  k_eig_prep / k_eig_finish (1184 x 256)           a level of > 303 104 nodes
  k_leaf_dist / k_leaf_pick (2368 x 256)           a leaf that owns a position >= 606 208
  scan_tile_sums_body, second pass                 > 2^20 points (level split, leaf starts) or records (compaction)
  k_decide_scan, second pass                       a level of > 2^20 nodes
  k_map_sums, second pass                          one map insert of > 1 047 552 points
  lane regrowth and level-graph re-capture         a batch larger than the lane (ensure_state: 2^17, then doubling)

Every case asserts, from the host tree's level widths and node sizes or from the record counts, that its input
crosses the thresholds it is there for, so that a change to a fixture cannot silently drop the coverage.  The CPU
test at the end checks the entry points' size-limit messages without a device."""
import ctypes as C
import os
import time

import numpy as np
import pytest

from mad_icp_b200 import FlatTree, MadIcpError, Registrar, _capi, records, synth
from test_gpu_tree_build import _same_as_oracle
from test_gpu_voxel_map import KITTI_GATE, MapOracle
from util import bits_equal

gpu = pytest.mark.gpu

LANE0 = 1 << 17            # the build lane's first capacity (ensure_state)
CLOUD_MAX = 1 << 24        # points per cloud
BATCH_MAX = 1 << 26        # points per batch
BIG_BLOCKS, BIG_NODE = 1776, 512
DECIDE = 64 * 1024
EIG = 1184 * 256
LEAF = 2368 * 256
TWO_PASS = 1 << 20         # 1024 tiles of 1024: past this, a tile-sum scan takes a second pass
MAP_ONE_PASS = 1023 * 1024  # k_map_sums scans n_tiles + 1 totals


# ----------------------------------------------------------------------------------------------------------- helpers
def _levels(recs, lo0):
    """per breadth-first level of a host tree's records (siblings adjacent): num_points, leaf flag and first point
    position of every node, the tree's points starting at position lo0 of the forest"""
    link, npts = recs["link"], recs["num_points"].astype(np.int64)
    lo = np.zeros(recs.shape[0], np.int64)
    lo[0] = lo0
    out, a, b = [], 0, 1
    while a < b:
        inner = np.flatnonzero(link[a:b] >= 0) + a
        kids = link[inner]
        lo[kids] = lo[inner]                      # the left child keeps the front of its parent's range
        lo[kids + 1] = lo[inner] + npts[kids]
        out.append((npts[a:b], link[a:b] < 0, lo[a:b]))
        a, b = b, b + 2 * inner.size
    return out


def _coverage(recs_list):
    """which second iterations a device build of the forest of these host trees runs (the table above); a forest level
    holds the trees' levels one after the other, in tree order"""
    offs = np.cumsum([0] + [int(r["num_points"][0]) for r in recs_list])
    per = [_levels(r, int(o)) for r, o in zip(recs_list, offs)]
    lv = []
    for d in range(max(len(p) for p in per)):
        parts = [p[d] for p in per if d < len(p)]
        lv.append(tuple(np.concatenate(x) for x in zip(*parts)))
    widths = [p.size for p, _, _ in lv]
    n = int(offs[-1])
    return dict(n=n, widest=max(widths),
                sums_big=any((p[BIG_BLOCKS:] >= BIG_NODE).any() for p, _, _ in lv[1:]),
                decide=max(widths) > DECIDE,
                eig=max(widths) > EIG,
                leaf=any(((lo + p)[leaf] > LEAF).any() for p, leaf, lo in lv),
                split=n > TWO_PASS,
                decide_scan=max(widths) > TWO_PASS)


def _same_records(dt, h):
    """a device tree's 64-byte records are the host builder's, byte for byte (NaN payloads aside)"""
    d = dt.records()
    assert dt.num_nodes == h.shape[0]
    for k in ("mean", "dir", "bbox0"):
        assert bits_equal(d[k], h[k]), f"{k}: {(~((d[k] == h[k]) | (np.isnan(d[k]) & np.isnan(h[k])))).sum()} differ"
    assert (d["link"] == h["link"]).all() and (d["num_points"] == h["num_points"]).all()


def _cloud(n, seed, extent=(40.0, 20.0, 3.0)):
    rs = np.random.RandomState(seed)
    return rs.uniform(0.0, 1.0, (n, 3)) * np.asarray(extent)


def _kitti(p, seed):
    """KITTI float32 N x 4 records of a scan with NaN rows, points nearer than 0.7 m and farther than 120 m among them"""
    rs = np.random.RandomState(seed)
    p = p.copy()
    rows = rs.choice(p.shape[0], 600, replace=False)
    p[rows[:300]] *= 0.01
    p[rows[300:]] *= 1.0e3
    p = np.insert(p, np.sort(rs.randint(0, p.shape[0], size=p.shape[0] // 20)), np.nan, axis=0)
    a = np.zeros((p.shape[0], 4), np.float32)
    a[:, :3] = p
    a[:, 3] = 0.5
    return a


@pytest.fixture(scope="module")
def seq40(built):
    """the bench's stream workload in small: 40 scans of 64 x 2048 along the street"""
    return synth.sequence(n_scans=40, beams=64, azimuths=2048)["scans"]


# ----------------------------------------------------------------------------------------------------------- GPU
@gpu
def test_lane_boundaries_in_one_context(oracle):
    """A full lane (2^17 points), its first regrowth (2^17 + 1) and a small cloud after it, in one context: the lane and
    the level graph captured for it are rebuilt at the regrowth and reused after it.  Then a batch larger than the lane
    while clouds are staged: the lane is re-allocated and the early uploads are given up."""
    reg = Registrar(device=0, max_keyframes=2)
    try:
        for n, seed in ((LANE0, 1), (LANE0 + 1, 2), (5000, 3)):
            cloud = _cloud(n, seed)
            dt = reg.build_tree(cloud)
            _same_as_oracle(dt, oracle.OracleTree(cloud), FlatTree(cloud))
        lane = 2 * LANE0  # after the regrowth
        staged = [_cloud(50000, 4), _cloud(60000, 5)]
        big = _cloud(200000, 6)
        batch = staged + [big]
        assert sum(c.shape[0] for c in staged) <= lane < sum(c.shape[0] for c in batch)
        want = [FlatTree(c).records() for c in batch]
        for c in staged:
            reg.stage_cloud(c)
        for dt, h in zip(reg.build_trees(batch), want):
            _same_records(dt, h)
        for c in staged:  # the grown lane holds the staged prefix: the early uploads are used
            reg.stage_cloud(c, sum(x.shape[0] for x in batch))
        for dt, h in zip(reg.build_trees(batch), want):
            _same_records(dt, h)
        dt = reg.build_tree(staged[0])
        _same_records(dt, want[0])
    finally:
        reg.close()


@gpu
def test_dense_cloud_past_a_million_nodes_per_level(oracle):
    """2^21 uniform points at b_max = b_min = 1e-5: a level of more than 2^20 nodes, and with it every second
    iteration of the level loop"""
    cloud = np.random.RandomState(21).uniform(0.0, 1.0, (1 << 21, 3))
    ft = FlatTree(cloud, b_max=1e-5, b_min=1e-5)
    cov = _coverage([ft.records()])
    assert all(cov[k] for k in ("sums_big", "decide", "eig", "leaf", "split", "decide_scan")), cov
    reg = Registrar(device=0, max_keyframes=2)
    try:
        dt = reg.build_tree(cloud, b_max=1e-5, b_min=1e-5)
        _same_as_oracle(dt, oracle.OracleTree(cloud, b_max=1e-5, b_min=1e-5), ft)
    finally:
        reg.close()


@gpu
def test_the_bench_forest(seq40):
    """32 scans of 64 x 2048 as one forest (Pipeline.prefetch's batch): float64 and float32 clouds, and KITTI records
    through the range gate, whose compaction scans more than 2^20 records"""
    scans = seq40[:32]
    want = [FlatTree(s).records() for s in scans]
    cov = _coverage(want)
    assert all(cov[k] for k in ("sums_big", "decide", "eig", "leaf", "split")), cov
    reg = Registrar(device=0, max_keyframes=2)
    try:
        for dt, h in zip(reg.build_trees(scans), want):
            _same_records(dt, h)
        f32 = [s.astype(np.float32) for s in scans]
        for dt, s in zip(reg.build_trees(f32), f32):
            _same_records(dt, FlatTree(s.astype(np.float64)).records())
        recs = [_kitti(s, seed=k) for k, s in enumerate(scans)]
        assert sum(a.shape[0] for a in recs) > TWO_PASS
        reg.keep_cloud(True)
        trees = reg.build_trees_records(recs, **KITTI_GATE)
        for a, dt in zip(recs, trees):
            mask = records.range_mask(a, **KITTI_GATE).astype(bool)
            kept = a[mask, :3].astype(np.float64)
            assert np.isnan(a[:, 0]).any() and 0 < mask.sum() < a.shape[0] - a.shape[0] // 25
            xyz, idx = dt.cloud()
            assert idx.shape[0] == mask.sum() and (idx == np.flatnonzero(mask)).all()
            assert bits_equal(xyz, kept)
            _same_records(dt, FlatTree(kept).records())
    finally:
        reg.close()


@gpu
def test_the_per_cloud_limit(oracle, seq40):
    """One cloud of exactly 2^24 points (every lane buffer exactly full), and the rejections past the limits: a cloud
    of 2^24 + 1 points through every entry, and a batch of more than 2^26 points before anything is allocated"""
    import torch
    assert all(s.shape[0] == LANE0 for s in seq40)  # (every ray of a scan in the street canyon hits)
    reg = Registrar(device=0, max_keyframes=2)
    try:
        def free():
            torch.cuda.synchronize()
            return torch.cuda.mem_get_info(0)[0]

        over = np.zeros((CLOUD_MAX + 1, 3))
        before = free()
        with pytest.raises(MadIcpError, match=r"1 <= n <= 2\^24"):
            reg.build_tree(over)
        with pytest.raises(MadIcpError, match=r"a cloud of more than 2\^24 points"):
            reg.build_trees([over])
        with pytest.raises(MadIcpError, match=r"1\.\.2\^24 records"):
            reg.build_trees_records([np.zeros((CLOUD_MAX + 1, 4), np.float32)], **KITTI_GATE)
        del over
        part = np.zeros((TWO_PASS + 1, 3))
        assert 64 * part.shape[0] > BATCH_MAX
        with pytest.raises(MadIcpError, match=r"more than 2\^26 points in the batch"):
            reg.build_trees([part] * 64)
        with pytest.raises(MadIcpError, match=r"more than 2\^26 points in the batch"):
            reg.build_trees_records([np.zeros((TWO_PASS + 1, 4), np.float32)] * 64, **KITTI_GATE)
        del part
        assert before - free() < 1 << 30  # a lane for these would take tens of GB

        # 128 scans side by side, 500 m apart: a city block of 2^24 points
        cloud = np.concatenate([seq40[k % 32] + [500.0 * (k // 32), 500.0 * (k % 32), 0.0] for k in range(128)])
        assert cloud.shape[0] == CLOUD_MAX
        t0 = time.perf_counter()
        ft = FlatTree(cloud)
        t_flat = time.perf_counter() - t0
        base = free()
        t0 = time.perf_counter()
        dt = reg.build_tree(cloud)
        used = base - free()
        t_dev = time.perf_counter() - t0
        cov = _coverage([ft.records()])
        assert all(cov[k] for k in ("sums_big", "decide", "eig", "leaf", "split")), cov
        _same_records(dt, ft.records())
        t0 = time.perf_counter()
        _same_as_oracle(dt, oracle.OracleTree(cloud), ft)
        print(f"\n2^24-point build: device memory of the lane and the tree {used / 2**30:.2f} GiB, {dt.num_nodes} nodes, "
              f"device {t_dev:.1f} s, FlatTree {t_flat:.1f} s, OracleTree and compare {time.perf_counter() - t0:.1f} s")
    finally:
        reg.close()


@gpu
@pytest.mark.parametrize("K", [1, 4])
def test_voxel_map_one_big_insert(K):
    """Inserts of 1 047 552 points (one k_map_sums pass), 1 047 553 and more than 2^21 (two passes), each with a second
    insert on top, into maps whose table grows past 2^22 slots"""
    v = 0.25
    reg = Registrar(device=0, max_keyframes=2)
    try:
        reg.keep_cloud(True)
        rs = np.random.RandomState(5)
        top = _cloud(700000, 50, extent=(64.0, 64.0, 64.0))
        clouds, trees = [], []
        for n in (MAP_ONE_PASS, MAP_ONE_PASS + 1, (1 << 21) + 4321):
            c = _cloud(n, n % 97, extent=(64.0, 64.0, 64.0))
            rows = rs.choice(n, 40, replace=False)
            c[rows[:20], 0] = 1.0e6  # keys out of range
            c[rows[20:], 1] = np.nan
            clouds.append(c)
            trees.append(reg.build_tree(c))
        t_top = reg.build_tree(top)
        T = synth.pose_xyyaw(1.3, -0.7, 0.2, z=0.4)
        X = np.asarray(T)[:3]
        top_map = ((X[None, :, 0] * top[:, 0:1] + X[None, :, 1] * top[:, 1:2]) + X[None, :, 2] * top[:, 2:3]) + X[None, :, 3]
        for c, t in zip(clouds, trees):
            o = MapOracle(v, K)
            o.insert(c, 3, np.arange(c.shape[0]))
            o.insert(top_map, 4, np.arange(top.shape[0]))
            m = reg.voxel_map(v, K)
            m.insert(t, None, scan=3)
            m.insert(t_top, T, scan=4)
            xyz, sr = m.points()
            want_xyz, want_sr = o.points()
            assert m.size() == want_xyz.shape[0] and m.dropped() == o.dropped == 40
            assert bits_equal(xyz, want_xyz) and (sr == want_sr).all()
            if c.shape[0] > 1 << 21:
                assert o.keys.size > 1 << 21  # load <= 1/2: more than 2^22 slots
            if K > 1:
                assert (o.counts > 1).any()  # voxels that took more than one point
            m.free()
    finally:
        reg.close()


@gpu
def test_bench_configuration_end_to_end(seq40):
    """The stream workload's configuration: look-ahead batches of 32 scans of 64 x 2048, no deskew, kept clouds and
    the map on.  Poses, keyframe decisions and inlier ratios are those of host-built trees bit for bit, and the map is
    the oracle's of the clouds the pipeline hands back."""
    from mad_icp_b200.pybind.pypeline import Pipeline
    kw = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=16,
              num_threads=min(16, os.cpu_count() or 1), realtime=False)

    def pipeline(gpu_build, **extra):
        os.environ["MADICP_GPU_BUILD"] = "1" if gpu_build else "0"
        try:
            return Pipeline(**kw, **extra)
        finally:
            os.environ.pop("MADICP_GPU_BUILD")

    scans, depth = seq40, 32
    assert sum(s.shape[0] for s in scans[1:1 + depth]) > TWO_PASS
    dev = pipeline(True, keep_cloud=True, map_voxel_size=0.2, map_points_per_voxel=2)
    host = pipeline(False)
    assert dev.gpuBuild() and not host.gpuBuild()
    o = MapOracle(0.2, 2)
    promoted = 0
    for i, scan in enumerate(scans):
        sid = dev.currentID()
        dev.compute(0.1 * i, scan)
        host.compute(0.1 * i, scan)
        if i == 0:
            for k in range(1, 1 + depth):
                assert dev.prefetch(scans[k])
        elif i + depth < len(scans):
            assert dev.prefetch(scans[i + depth])
        o.insert(dev.currentCloudArray(frame="map"), sid, dev.currentCloudIndices())
        assert bits_equal(dev.currentPose(), host.currentPose()), i
        assert (dev.isMapUpdated(), dev.keyframeID(), dev.numKeyframes()) == \
            (host.isMapUpdated(), host.keyframeID(), host.numKeyframes()), i
        assert dev.inliersRatio() == host.inliersRatio(), i
        promoted += int(dev.isMapUpdated())
    assert promoted >= 3
    want_xyz, want_sr = o.points()
    assert dev.mapSize() == want_xyz.shape[0] > 0 and dev.mapDropped() == o.dropped
    assert bits_equal(dev.mapArray(), want_xyz) and (dev.mapIndices() == want_sr).all()


# ----------------------------------------------------------------------------------------------------------- no GPU
def test_size_limit_messages_without_gpu(built):
    """The per-cloud limit (2^24) and the per-batch limit (2^26) are named by the entry points that enforce them,
    before the context is touched (the fake one below is never dereferenced) and before a point is read"""
    L = _capi.lib()
    fake = C.c_void_p(1)
    buf = np.zeros((4, 4), np.float32)
    out = (C.c_void_p * 64)()
    ptrs = (C.c_void_p * 64)(*([buf.ctypes.data] * 64))
    ns = (C.c_int64 * 64)(CLOUD_MAX + 1)
    assert L.madtree_gpu_build_batch(fake, ptrs, ns, 0, 1, 0.2, 0.1, out) == -1
    assert L.madicp_last_error() == b"madtree_gpu_build_batch: empty cloud, or a cloud of more than 2^24 points"
    ns = (C.c_int64 * 64)(*([TWO_PASS + 1] * 64))
    assert L.madtree_gpu_build_batch(fake, ptrs, ns, 0, 64, 0.2, 0.1, out) == -1
    assert b"madtree_gpu_build_batch: more than 2^26 points in the batch" in L.madicp_last_error()
    assert L.madtree_gpu_build(fake, _capi.as_d(buf.astype(np.float64)), CLOUD_MAX + 1, 0.2, 0.1, C.byref(C.c_void_p())) == -1
    assert b"1 <= n <= 2^24" in L.madicp_last_error()
    d = records.describe(buf, **KITTI_GATE)
    d.n = CLOUD_MAX + 1
    descs = (_capi.Points * 64)(*([d] * 64))
    assert L.madtree_gpu_build_batch_points_ex(fake, descs, None, 1, 0.2, 0.1, out) == -1
    assert b"n must be 1..2^24 records" in L.madicp_last_error()
    d.n = TWO_PASS + 1
    descs = (_capi.Points * 64)(*([d] * 64))
    assert L.madtree_gpu_build_batch_points_ex(fake, descs, None, 64, 0.2, 0.1, out) == -1
    assert b"madtree_gpu_build_batch_points: more than 2^26 points in the batch" in L.madicp_last_error()
