"""MAD-tree build and scan ingest ON THE DEVICE (SURVEY 8f next-1 / next-3), `-m gpu`: the device-built tree must be
the reference's tree node for node and bit for bit -- topology, means, all nine eigenvector coefficients (including
the NaNs of one-point nodes), bounding boxes, point counts, leaf order -- against the CPU oracle (which is pinned to
the reference's own sources, tests/test_reference_pin.py) and against the host builder; registration from a
device-built tree must give the same bits as from a host-built one; the device ingest must reproduce
Pipeline::deskew (odometry/pipeline.cpp:79-123) bit for bit."""
import numpy as np
import pytest

from mad_icp_b200 import FlatTree, Registrar, synth
from util import bits_equal

pytestmark = pytest.mark.gpu


def _bfs_order(e):
    """DFS pre-order export (left/right node ids) -> node ids in breadth-first order, siblings adjacent."""
    order, level = [], np.zeros(1, np.int64)
    while level.size:
        order.append(level)
        inner = level[e["left"][level] >= 0]
        level = np.stack([e["left"][inner], e["right"][inner]], 1).ravel().astype(np.int64)
    return np.concatenate(order)


def _same_as_oracle(dt, otree, ft=None):
    e = otree.export()
    order = _bfs_order(e)
    d = dt.export()
    assert dt.num_nodes == len(order) and dt.num_leaves == otree.num_leaves
    for k in ("mean", "eivecs", "bbox"):
        assert bits_equal(d[k], e[k][order]), f"{k}: {(d[k] != e[k][order]).sum()} coefficients differ (NaN-aware compare failed)"
    assert (d["num_points"] == e["num_points"][order]).all()
    recs = dt.records()
    leaf = recs["link"] < 0
    assert ((-1 - recs["link"][leaf]) == e["leaf_ordinal"][order][leaf]).all()
    assert (e["leaf_ordinal"][order][~leaf] == -1).all()
    if ft is not None:  # and the 64-byte records are the host builder's, byte for byte (NaN payloads aside)
        h = ft.records()
        for k in ("mean", "dir", "bbox0"):
            assert bits_equal(recs[k], h[k]), k
        assert (recs["link"] == h["link"]).all() and (recs["num_points"] == h["num_points"]).all()


@pytest.fixture(scope="module")
def reg():
    return Registrar(device=0, max_keyframes=4)


@pytest.mark.parametrize("beams,azimuths,seed", [(16, 512, 3), (32, 1024, 5), (64, 2048, 1)])
def test_lidar_scan_tree_is_the_references(reg, oracle, beams, azimuths, seed):
    c = synth.registration_case(K=1, beams=beams, azimuths=azimuths, seed=seed)
    for cloud in (c["scans"][0], c["query"]):
        dt = reg.build_tree(cloud)
        _same_as_oracle(dt, oracle.OracleTree(cloud), FlatTree(cloud))


@pytest.mark.parametrize("b_max,b_min", [(0.2, 0.1), (0.05, 0.02), (1e-5, 0.1), (1.0, 0.5)])
def test_four_walls_and_parameters(reg, oracle, b_max, b_min):
    np.random.seed(42)
    cloud = synth.four_walls(points_per_wall=2000 if b_max < 1e-3 else 4000)
    dt = reg.build_tree(cloud, b_max=b_max, b_min=b_min)
    _same_as_oracle(dt, oracle.OracleTree(cloud, b_max=b_max, b_min=b_min), FlatTree(cloud, b_max=b_max, b_min=b_min))


def test_degenerate_clouds(reg, oracle):
    rs = np.random.RandomState(0)
    clouds = [np.array([[1.0, 2.0, 3.0]]),                                   # one point: NaN covariance, root leaf
              np.array([[0.0, 0, 0], [1.0, 0, 0]]),                          # two points
              np.repeat(np.array([[0.5, -1.0, 2.0]]), 50, axis=0),            # all identical
              np.stack([np.linspace(0, 10, 200), np.zeros(200), np.zeros(200)], 1),   # collinear
              np.concatenate([rs.normal(0, 0.01, (300, 3)), rs.normal(5, 0.01, (3, 3)), [[9.0, 9, 9]]]),  # tiny clusters
              rs.uniform(-1, 1, (1000, 3)) * [10, 10, 0]]                   # planar
    for cloud in clouds:
        dt = reg.build_tree(cloud)
        _same_as_oracle(dt, oracle.OracleTree(cloud), FlatTree(cloud))


def test_batch_build_is_a_forest_of_the_same_trees(reg, oracle):
    """madtree_gpu_build_batch: several scans built as one forest must give, tree for tree, the records of the single
    builds (and hence the reference's), for ragged batches (different sizes, a one-point cloud, planar clouds)."""
    c = synth.registration_case(K=3, beams=32, azimuths=1024, seed=21)
    rs = np.random.RandomState(1)
    clouds = [c["scans"][0], c["scans"][1][:5000], np.array([[1.0, 2.0, 3.0]]), c["query"],
              rs.uniform(-1, 1, (700, 3)) * [10, 10, 0], c["scans"][2]]
    trees = reg.build_trees(clouds)
    for cloud, dt in zip(clouds, trees):
        ft = FlatTree(cloud)
        h, d = ft.records(), dt.records()
        assert dt.num_nodes == ft.num_nodes and dt.num_leaves == ft.num_leaves and dt.num_levels == len(_bfs_levels(h))
        for k in ("mean", "dir", "bbox0"):
            assert bits_equal(d[k], h[k]), k
        assert (d["link"] == h["link"]).all() and (d["num_points"] == h["num_points"]).all()
        leaf = np.nonzero(h["link"] < 0)[0]
        want = np.empty(ft.num_leaves, np.int32)
        want[-1 - h["link"][leaf]] = leaf
        assert (dt.leaf_records() == want).all()
    f32 = [cl.astype(np.float32) for cl in clouds[:3]]
    for cloud, dt in zip(f32, reg.build_trees(f32)):
        assert dt.records().tobytes() == FlatTree(cloud.astype(np.float64)).records().tobytes() or \
            bits_equal(dt.records()["mean"], FlatTree(cloud.astype(np.float64)).records()["mean"])


def test_staged_clouds_build_the_same_forest(reg, oracle):
    """madicp_stage_cloud: early uploads change where the copy happens, never the trees: a full prefix, a partial one,
    a staged cloud the batch does not start with, and a single build in between (which discards what was staged)."""
    c = synth.registration_case(K=3, beams=32, azimuths=1024, seed=23)
    clouds = [np.ascontiguousarray(x) for x in (c["scans"][0], c["scans"][1][:7000], c["query"], c["scans"][2])]
    want = [FlatTree(cl).records() for cl in clouds]

    def same(d, h):
        return all(bits_equal(d[k], h[k]) for k in ("mean", "dir", "bbox0")) and (d["link"] == h["link"]).all() and \
            (d["num_points"] == h["num_points"]).all()

    def check(trees, idx):
        for dt, i in zip(trees, idx):
            assert same(dt.records(), want[i]), i

    total = sum(cl.shape[0] for cl in clouds)
    for cl in clouds:  # everything staged, in order
        reg.stage_cloud(cl, total)
    check(reg.build_trees(clouds), range(4))
    for cl in clouds[:2]:  # a prefix only
        reg.stage_cloud(cl, total)
    check(reg.build_trees(clouds), range(4))
    reg.stage_cloud(clouds[1], total)  # staged, but the batch starts with another cloud
    reg.stage_cloud(clouds[0], total)
    check(reg.build_trees([clouds[0], clouds[1], clouds[3]]), [0, 1, 3])
    reg.stage_cloud(clouds[2], total)  # a single build in between discards the staged cloud
    assert same(reg.build_tree(clouds[3]).records(), want[3])
    check(reg.build_trees([clouds[2], clouds[0]]), [2, 0])
    f32 = [np.ascontiguousarray(cl[:3000].astype(np.float32)) for cl in clouds[:3]]
    for cl in f32:
        reg.stage_cloud(cl, 9000)
    for cl, dt in zip(f32, reg.build_trees(f32)):
        assert same(dt.records(), FlatTree(cl.astype(np.float64)).records())
    reg.stage_cloud(f32[0], 0)  # float32 staged, float64 batch
    check(reg.build_trees(clouds[:2]), [0, 1])
    # staged, then given up (madicp_stage_discard): the buffers may go away at once, the next batch is unaffected
    gone = [cl.copy() for cl in clouds[:2]]
    for cl in gone:
        reg.stage_cloud(cl, total)
    reg.stage_discard()
    for cl in gone:
        cl[:] = np.nan
    del gone
    reg.stage_discard()  # nothing staged: a no-op
    check(reg.build_trees(clouds), range(4))


def _bfs_levels(recs):
    """level sizes of breadth-first records with adjacent siblings"""
    sizes, lo, hi = [], 0, 1
    while lo < hi:
        sizes.append(hi - lo)
        links = recs["link"][lo:hi]
        nxt = 2 * int((links >= 0).sum())
        lo, hi = hi, hi + nxt
    return sizes


def test_registration_from_device_built_trees(reg):
    """The whole device-resident chain: build on the device -> moving leaves from the device tree -> promotion with the
    pose applied on the device; same bits as host-built trees transformed on the host."""
    c = synth.registration_case(K=3, beams=32, azimuths=1024, seed=11)
    a = Registrar(device=0, max_keyframes=4)
    for k, (scan, P) in enumerate(zip(c["scans"], c["kf_poses"])):
        ft = FlatTree(scan)
        ft.apply_transform(P)
        a.put_keyframe(k, ft)
        reg.put_keyframe(k, reg.build_tree(scan), T=P)
    q = FlatTree(c["query"])
    a.set_moving(q.leaf_means())
    reg.set_moving_tree(reg.build_tree(c["query"]))
    assert bits_equal(reg.get_moving(), q.leaf_means())
    assert (a.search(c["T_guess"]) == reg.search(c["T_guess"])).all()
    ra, rb = a.register(c["T_guess"], iters=10), reg.register(c["T_guess"], iters=10)
    for k in ("X", "H", "b"):
        assert bits_equal(ra[k], rb[k]), k
    assert (ra["matched"] == rb["matched"]).all()
    for k in range(3):
        reg.drop_keyframe(k)


def test_ingest_float32_and_deskew(reg, oracle):
    c = synth.registration_case(K=1, beams=32, azimuths=1024, seed=8)
    cloud = c["query"]
    f32 = cloud.astype(np.float32)
    out = reg.ingest(f32, want_points=True)
    assert bits_equal(out, f32.astype(np.float64))                 # the readers' float32 -> float64 (exact)
    dt = reg.build_tree()                                          # tree of the cloud the ingest left on the device
    _same_as_oracle(dt, oracle.OracleTree(f32.astype(np.float64)))
    # deskew: against the CPU pipeline's (itself pinned to the reference's Pipeline::deskew)
    T_prev = synth.pose_xyyaw(0.0, 0.0, 0.0)
    T_now = synth.pose_xyyaw(0.8, 0.05, 0.02)
    want = oracle.deskew(cloud, T_prev, T_now, sensor_hz=10.0)
    for threads in (1, 4):
        got = reg.ingest(cloud, deskew=True, T_prev=T_prev, T_now=T_now, sensor_hz=10.0, num_threads=threads, want_points=True)
        assert bits_equal(got, want), f"{threads} threads: {(got != want).any(axis=1).sum()} points differ"
    # tied azimuths (noise-free rings: whole firing columns share an azimuth) and float32 input
    az = np.repeat(np.linspace(-np.pi, np.pi, 256, endpoint=False), 16)
    r = np.tile(np.linspace(2.0, 30.0, 16), 256)
    tied = np.stack([r * np.cos(az), r * np.sin(az), np.tile(np.linspace(-2, 1, 16), 256)], 1).astype(np.float32)
    want = oracle.deskew(tied.astype(np.float64), T_prev, T_now, sensor_hz=10.0)
    got = reg.ingest(tied, deskew=True, T_prev=T_prev, T_now=T_now, sensor_hz=10.0, num_threads=2, want_points=True)
    assert bits_equal(got, want)


def test_pipeline_device_path_lookahead_and_host_path_agree(oracle):
    """The reference-named Pipeline three ways -- trees built on the device in line, trees built ahead of time by the
    look-ahead lanes (Pipeline.prefetch), trees built on the host (MADICP_GPU_BUILD=0) -- must produce bit-identical
    trajectories and keyframe decisions (same trees, same registration), and track the CPU pipeline."""
    import os
    from mad_icp_b200.pybind.pypeline import Pipeline
    seq = synth.sequence(n_scans=20, beams=32, azimuths=1024, seed=4)["scans"]
    kw = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
              num_threads=4, realtime=False)

    def run(mode):
        os.environ["MADICP_GPU_BUILD"] = "0" if mode == "host" else "1"
        p = Pipeline(**kw)
        os.environ.pop("MADICP_GPU_BUILD")
        assert p.gpuBuild() == (mode != "host")
        out = []
        for i, scan in enumerate(seq):
            if mode == "lookahead" and i >= 1 and p.prefetched() == 0:
                # compute() consumes prefetched scans in FIFO order: hand over the next five (one forest build)
                for k in range(i, min(i + 5, len(seq))):
                    assert p.prefetch(seq[k])
            p.compute(0.1 * i, scan)
            out.append((p.currentPose().copy(), bool(p.isMapUpdated()), int(p.keyframeID()), int(p.numKeyframes())))
        return out

    a, b, c = run("inline"), run("lookahead"), run("host")
    cpu = oracle.OraclePipeline(**kw)
    promoted = 0
    for i, scan in enumerate(seq):
        cpu.compute(0.1 * i, scan)
        st = cpu.state()
        for other in (b, c):
            assert bits_equal(a[i][0], other[i][0]), i
            assert a[i][1:] == other[i][1:], i
        assert a[i][1:] == (bool(st[12]), int(st[14]), int(st[15])), i
        assert np.abs(a[i][0][:3] - st[:12].reshape(3, 4)).max() < 1e-6, i
        promoted += int(st[12])
    assert promoted >= 3


def test_pipeline_realtime_budget(oracle):
    """`realtime` (pipeline.cpp:62,167-169): the sensor period minus 5 ms minus the preprocessing time bounds the
    rounds.  A generous period never binds (bit-identical to the unbounded pipeline, 15 rounds); a period shorter than
    the preprocessing alone leaves no round at all -- the reference breaks out of its loop at iteration 0 too -- and the
    pose stays the constant-velocity prediction."""
    from mad_icp_b200.pybind.pypeline import Pipeline
    seq = synth.sequence(n_scans=8, beams=32, azimuths=1024, seed=4)["scans"]
    kw = dict(deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4, num_threads=4)
    free = Pipeline(sensor_hz=10.0, realtime=False, **kw)
    slack = Pipeline(sensor_hz=10.0, realtime=True, **kw)    # 95 ms budget: never binds on a GPU
    tight = Pipeline(sensor_hz=199.0, realtime=True, **kw)   # 1000/199 - 5 = 0.025 ms: less than any preprocessing
    for i, scan in enumerate(seq):
        for p in (free, slack, tight):
            p.compute(0.1 * i, scan)
        assert bits_equal(free.currentPose(), slack.currentPose()), i
        if i > 0:
            assert slack.lastIcpIterations() == 15 and tight.lastIcpIterations() == 0
        assert np.isfinite(tight.currentPose()).all()
    assert np.abs(tight.currentPose() - np.eye(4)).max() == 0.0  # never registered: identity + zero velocity
