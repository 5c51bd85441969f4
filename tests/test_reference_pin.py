"""Pins the CPU restatement (oracle/) against the reference's OWN sources.

tests/golden/reference_pin.json holds SHA-256 digests (tests/util.py: digest) of every array the reference computed
for the cases below: tools/mad_tree.cpp, odometry/mad_icp.cpp, odometry/vel_estimator.cpp and odometry/pipeline.cpp
compiled unmodified against oracle/eigen_standin (`make -C oracle ref`) and run through the same case functions by
tests/golden/make_reference_pin.py.  Everything the reference decides -- split order, leaf selection, normal
inheritance, NaN handling of 1-point nodes, gate, kernel, accumulation order, keyframe promotion -- runs as written by
its authors; the restatement must reproduce it bit for bit, i.e. every array must hash to the reference's digest.
What stays unpinned is the evaluation order INSIDE Eigen's operators, which the stand-in takes from the restatement
(see its header).

CPU only; needs nothing outside the repository.
"""
import json
import os
import types

import numpy as np
import pytest

from mad_icp_b200 import synth
from util import digest

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_pin.json")


def backend(oracle_module):
    """The CPU restatement behind the interface the case functions use (make_reference_pin.py: reference_backend)."""
    O = oracle_module
    return types.SimpleNamespace(Tree=lambda pts, max_parallel_level=0, **kw: O.OracleTree(pts, **kw), icp_run=O.icp_run,
                                 Pipeline=O.OraclePipeline, deskew=O.deskew, idx_kw={})


def tree_arrays(t):
    out = dict(t.export())
    out["cloud"] = t.cloud()  # the build reorders and writes into the caller's vector
    out["shape"] = np.array([t.num_nodes, t.num_leaves])
    return out


def icp_arrays(r, with_idx=True):
    keys = ("X_hist", "H_hist", "b_hist", "X", "matched") + (("idx_hist",) if with_idx else ())
    return {k: np.asarray(r[k]) for k in keys}


# ---------------------------------------------------------------------------------------------- cases
# Every case maps a backend to {name: {key: array}}; the same functions produce the stored digests.
def case_tree_build(M, b_max):
    np.random.seed(42)
    cloud = synth.four_walls(points_per_wall=2000)
    return {"tree": tree_arrays(M.Tree(cloud, b_max=b_max))}


def case_lidar_scan_and_async_levels(M):
    """max_parallel_level > 0 takes the reference's std::async branch (mad_tree.cpp:106-128): same tree."""
    case = synth.registration_case(K=1, beams=32, azimuths=1024)
    pts = case["scans"][0]
    out = {f"level{lv}": tree_arrays(M.Tree(pts, max_parallel_level=lv)) for lv in (0, 3)}
    t = M.Tree(pts)
    t.apply_transform(case["kf_poses"][0])
    out["transformed"] = tree_arrays(t)
    out["search"] = {"idx": t.search(case["query"][:5000])}
    return out


def case_degenerate_clouds(M):
    rs = np.random.RandomState(3)
    clouds = (rs.rand(1, 3), rs.rand(2, 3), rs.rand(3, 3), np.repeat(rs.rand(1, 3), 50, axis=0),
              np.c_[rs.rand(200, 2), np.zeros(200)], np.c_[rs.rand(64), np.zeros((64, 2))])
    return {f"cloud{i}": tree_arrays(M.Tree(pts, b_max=0.05)) for i, pts in enumerate(clouds)}


def case_registration_loop(M, K, threads):
    case = synth.registration_case(K=K, beams=16, azimuths=512)
    kf = []
    for s in range(K):
        t = M.Tree(case["scans"][s])
        t.apply_transform(case["kf_poses"][s])
        kf.append(t)
    r = M.icp_run(kf, M.Tree(case["query"]), case["T_guess"], iters=10, num_threads=threads, **M.idx_kw)
    # idx_hist: the correspondences themselves, the reference's bestMatchingLeafFast on its own X_ * mean_, every round
    return {"icp": icp_arrays(r)}


def case_four_walls_demo(M):
    """apps/utils/tools/mad_registration.py: 15 poses and H/b, converging to identity."""
    np.random.seed(42)
    cloud = synth.four_walls(points_per_wall=1000)
    T = np.eye(4)
    T[:3, :3] = synth.euler_xyz(0.1, 0.1, 0.1)
    T[:3, 3] = np.random.rand(3)
    return {"icp": icp_arrays(M.icp_run([M.Tree(cloud)], M.Tree(cloud), T, iters=15), with_idx=False)}


def _sequence(n, beams=16, azimuths=512):
    scene = synth.StreetScene(seed=7)
    for i in range(n):
        base = synth.pose_xyyaw(0.8 * i, 1.0 + 0.02 * i, 0.004 * i)
        yield 0.1 * i, np.ascontiguousarray(synth.lidar_scan(scene, base, beams=beams, azimuths=azimuths, seed=100 + i))


def case_pipeline(M, deskew):
    """Streaming odometry: pose (frame_to_map_), map updated / ids / number of keyframes and the VelEstimator state of
    every scan.  (The keyframe weight det(H^-1), column 16, is computed by two independently written LU routines; only
    the decisions it drives are compared.)"""
    p = M.Pipeline(deskew=deskew, num_keyframes=4, num_threads=4)
    st = []
    for stamp, pts in _sequence(16):
        p.compute(stamp, pts)
        st.append(p.state())
    st = np.array(st)
    return {"state": {"pose": st[:, :12], "keyframes": st[:, 12:16], "velocity": st[:, 17:]}}


def case_deskew(M):
    _, pts = next(_sequence(1))
    Ta, Tb = synth.pose_xyyaw(0.0, 1.0, 0.0), synth.pose_xyyaw(0.8, 1.05, 0.03)
    return {"deskew": {"points": M.deskew(pts, Ta, Tb)}}


def case_parameter_sweep(M, b_max, b_min, rho_ker, b_ratio):
    """Other leaf sizes, kernel widths and gate ratios than the defaults: trees and every GN round."""
    case = synth.registration_case(K=2, beams=16, azimuths=512, seed=9)
    out, kf = {}, []
    for s, (pts, P) in enumerate(zip(case["scans"], case["kf_poses"])):
        t = M.Tree(pts, b_max=b_max, b_min=b_min)
        out[f"tree{s}"] = tree_arrays(t)
        t.apply_transform(P)
        kf.append(t)
    mo = M.Tree(case["query"], b_max=b_max, b_min=b_min)
    r = M.icp_run(kf, mo, case["T_guess"], iters=6, min_ball=b_max, rho_ker=rho_ker, b_ratio=b_ratio, num_threads=2)
    out["icp"] = icp_arrays(r, with_idx=False)
    return out


# the last: a negative ratio makes every gate radius negative (|mean| > 4 m for every leaf of the case), and the
# reference's `norm > ball` then rejects every pair
SWEEP = [(0.1, 0.05, 0.05, 0.01), (0.4, 0.2, 0.3, 0.05), (0.2, 0.1, 1e-3, 0.0), (0.2, 0.1, 0.1, -0.05)]
CASES = {f"tree_build[{b}]": (case_tree_build, dict(b_max=b)) for b in (0.2, 1e-5)}
CASES["lidar_scan_and_async_levels"] = (case_lidar_scan_and_async_levels, {})
CASES["degenerate_clouds"] = (case_degenerate_clouds, {})
CASES.update({f"registration_loop[{K}-{t}]": (case_registration_loop, dict(K=K, threads=t)) for K, t in [(1, 1), (3, 2), (4, 4)]})
CASES["four_walls_demo"] = (case_four_walls_demo, {})
CASES.update({f"pipeline[{d}]": (case_pipeline, dict(deskew=d)) for d in (False, True)})
CASES["deskew"] = (case_deskew, {})
CASES.update({"parameter_sweep[%g-%g-%g-%g]" % p: (case_parameter_sweep, dict(zip(("b_max", "b_min", "rho_ker", "b_ratio"), p)))
              for p in SWEEP})


def digests(out):
    return {part: {k: digest(v) for k, v in arrays.items()} for part, arrays in out.items()}


# ---------------------------------------------------------------------------------------------- tests
@pytest.fixture(scope="module")
def pinned():
    with open(GOLDEN) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def M(oracle):
    return backend(oracle)


def _run(M, pinned, name):
    fn, kw = CASES[name]
    out = fn(M, **kw)
    got, want = digests(out), pinned[name]
    assert set(got) == set(want), name
    for part in want:
        diff = [k for k in want[part] if got[part].get(k) != want[part][k]]
        assert not diff, f"{name}/{part}: {diff} differ from the reference's"
    return out


@pytest.mark.parametrize("b_max", [0.2, 1e-5])
def test_tree_build_is_the_references(M, pinned, b_max):
    _run(M, pinned, f"tree_build[{b_max}]")


def test_tree_build_lidar_scan_and_async_levels(M, pinned):
    _run(M, pinned, "lidar_scan_and_async_levels")


def test_degenerate_clouds(M, pinned):
    _run(M, pinned, "degenerate_clouds")


@pytest.mark.parametrize("K,threads", [(1, 1), (3, 2), (4, 4)])
def test_registration_loop_is_the_references(M, pinned, K, threads):
    _run(M, pinned, f"registration_loop[{K}-{threads}]")


def test_four_walls_demo_is_the_references(M, pinned):
    out = _run(M, pinned, "four_walls_demo")
    assert np.abs(out["icp"]["X"] - np.eye(4)[:3]).max() < 1e-6


@pytest.mark.parametrize("deskew", [False, True])
def test_pipeline_is_the_references(M, pinned, deskew):
    out = _run(M, pinned, f"pipeline[{deskew}]")
    assert int(out["state"]["keyframes"][:, 0].sum()) >= 4


def test_deskew_is_the_references(M, pinned):
    out = _run(M, pinned, "deskew")
    _, pts = next(_sequence(1))
    assert np.abs(out["deskew"]["points"] - pts).max() > 1e-3  # it did something


@pytest.mark.parametrize("b_max,b_min,rho_ker,b_ratio", SWEEP)
def test_parameter_sweep_is_the_references(M, pinned, b_max, b_min, rho_ker, b_ratio):
    out = _run(M, pinned, "parameter_sweep[%g-%g-%g-%g]" % (b_max, b_min, rho_ker, b_ratio))
    icp = out["icp"]
    if b_ratio < 0:  # the pinned digests are those of "nothing matched": H = b = 0, the pose never moves
        assert not icp["matched"].any()
        assert (icp["H_hist"] == 0).all() and (icp["b_hist"] == 0).all()
        assert (icp["X"] == icp["X_hist"][0]).all()
    else:
        assert icp["matched"].mean() > 0.5
