"""The product's Pipeline against the reference's own odometry/pipeline.cpp over the same device kernels, bit for bit.

oracle/_ref/libmadicp_ref_gpu.so is the reference's unmodified pipeline.cpp and vel_estimator.cpp linked with
mad_icp_b200/csrc/adapter/reference_backend.cpp: the same trees, the same persistent Gauss-Newton kernel and the same
keyframe slots as mad_icp_b200's Pipeline.  What differs is the host logic around them -- the velocity estimator and
the prediction, the frames window, the keyframe choice by det(H^-1), eviction, the inlier ratio and the slot
bookkeeping -- which pipeline.hpp and facade.hpp restate.  So the two must agree bit for bit on every scan, and any
difference is a host-side departure.  The looser bars of test_pybind_api.py / test_gpu_params.py (1e-5 rad, 1e-4 m
against the CPU oracle) cannot see one: 15 GN rounds pull a slightly wrong prediction back to the same pose.

1. The premise underneath: the backend runs one GN round per launch, Pipeline all of a scan's rounds in one.  Round k
   of a chained launch must equal a fresh one-round launch from the same pose -- poses, H/b, flags and weight.
2. Sequences that reach the branches a gentle lane never does: a speed step from rest (the velocity estimator's Huber
   scale), turns, a stationary stretch of one repeated scan array, pitch and roll, promotion on every scan and never.
   Each run asserts, through the probe of oracle/ref_capi.cpp, that it reached what it is meant to reach; where the
   CPU build of the reference (libmadicp_ref.so) reaches the same branches the asserts also run without a GPU.
3. Every scan of every run through Pipeline's routes -- plain float64 compute, look-ahead at depth 5 (deskew_ahead on
   deskewed runs), host-built trees (MADICP_GPU_BUILD=0), and keep_cloud with a voxel map -- against the reference
   run: pose, keyframe decision and pose, inlier ratio, the current and the model leaves; the trajectory at the end.

One deliberate departure is not compared: after the first scan the reference's currentLeaves() is empty (initialize
fills no current_leaves_), while Pipeline's current scan is the first one and currentLeaves() hands out its leaves
(DESIGN.md, "Pipeline against the reference").
"""
import functools
import gc
import hashlib
import os
from unittest import mock

import numpy as np
import pytest

from mad_icp_b200 import FlatTree, Registrar, synth
from test_gpu_params import PIPE_SETS
from test_gpu_rounds import PARAMS
from util import bits_equal

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HZ = 10.0
E_THRESHOLD_VEL = 0.3162  # tools/constants.h
FRAME_WINDOW = 10
MAX_ITERS = 64  # MADICP_MAX_ITERS: rounds per launch


# ------------------------------------------------------------------ sequences
def _scene():
    return synth.StreetScene(seed=7, x_max=120.0)


def _scans(poses, beams, azimuths, seed, replay=()):
    """Sensor-frame scans at the given base poses; scan i in `replay` is the same array object as scan i - 1 (a vehicle
    at a standstill whose sweep is handed over again)."""
    scene, out = _scene(), []
    for i, T in enumerate(poses):
        if i in replay:
            out.append(out[i - 1])
        else:
            out.append(synth.lidar_scan(scene, T, beams=beams, azimuths=azimuths, seed=seed + i))
    return out


def turns_and_stops(beams=32, azimuths=1024):
    """At rest for three scans of one replayed sweep: registered exactly where they started, two frames of identical
    weight, which the keyframe choice on leaving must tell apart the way pipeline.cpp:238-244 does (the first one).
    Then from rest to 1 m per scan in two scans (the velocity estimator meets errors far above its Huber threshold),
    a left and a right turn of up to 0.08 rad per scan, a stop, and five hand-overs of the same scan array."""
    v = [0.0, 0.0, 0.0, 0.5] + [1.0] * 12 + [0.6, 0.2, 0.0] + [0.0] * 5
    w = [0.0] * 6 + [0.08, 0.08, 0.06, 0.0, 0.0, -0.08, -0.08, -0.06] + [0.0] * 10
    T, poses = synth.pose_xyyaw(0.0, 1.0, 0.0), []
    for i in range(len(v)):
        T = T @ synth.pose_xyyaw(v[i], 0.0, w[i])
        poses.append(T.copy())
    return _scans(poses, beams, azimuths, seed=500, replay={1, 2} | set(range(len(v) - 5, len(v))))


def bumps(beams=32, azimuths=1024):
    """0.8 m per scan over a bumpy road: roll and pitch of a few degrees and a bouncing height, so every velocity
    component and the asin / atan2 terms of the estimator are non-trivial."""
    poses = []
    for i in range(18):
        T = synth.pose_xyyaw(0.8 * i, 1.0 + 0.2 * np.sin(0.4 * i), 0.03 * np.sin(0.5 * i), z=0.05 * np.sin(1.3 * i))
        R = np.eye(4)
        R[:3, :3] = synth.euler_xyz(0.05 * np.sin(0.9 * i), 0.06 * np.sin(0.7 * i + 0.5), 0.0)
        poses.append(T @ R)
    return _scans(poses, beams, azimuths, seed=700)


@functools.lru_cache(maxsize=None)
def sequence(name):
    if name == "turns":
        return tuple(turns_and_stops())
    if name == "bumps":
        return tuple(bumps())
    assert name == "lane64"  # the bench's shape: 64 x 2048 sweeps of the gentle lane
    return tuple(synth.sequence(n_scans=100, beams=64, azimuths=2048, workers=min(16, os.cpu_count() or 1))["scans"])


# (sequence, parameter set, num_keyframes, deskew, p_th override or None)
CONFIGS = (
    [(s, "default", k, d, None) for s in ("turns", "bumps") for k in (1, 4, 16) for d in (0, 1)]
    + [(s, p, 4, d, None) for s in ("turns", "bumps") for p in ("set0", "set1") for d in (0, 1)]
    + [("turns", "default", k, d, 1.0) for k in (1, 4) for d in (0, 1)]  # a promotion on every scan
    + [("turns", "default", 4, 0, 0.0), ("bumps", "default", 4, 1, 0.0)]  # no promotion after the first scan
)
BIG = ("lane64", "default", 16, 0, None)


def _cid(cfg):
    s, p, k, d, pth = cfg
    return f"{s}-{p}-kf{k}-deskew{d}" + ("" if pth is None else f"-pth{pth:g}")


def _kw(cfg):
    _, pset, k, d, pth = cfg
    b_max, b_min, rho_ker, p_th, b_ratio = (0.2, 0.1, 0.1, 0.8, 0.02) if pset == "default" else PIPE_SETS[int(pset[-1])]
    return dict(sensor_hz=HZ, deskew=bool(d), b_max=b_max, rho_ker=rho_ker, p_th=p_th if pth is None else pth, b_min=b_min,
                b_ratio=b_ratio, num_keyframes=k, num_threads=4, realtime=False)


# ------------------------------------------------------------------ the reference's run, through the probe
def _digest(a):
    return hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()


def reference_run(mod, cfg, leaves=True):
    """One pass of the reference's Pipeline (module `mod`: oracle.reference or a variant of it) over cfg's sequence:
    per scan the state, and through the probe the frames window, the keyframes and the leaves (the model's as a digest);
    the trajectory.  A library that predates the probe (mod.has_probe(), prebuilt where the reference sources are not
    at hand to rebuild it) yields the state alone: no inlier ratio, no lists, the trajectory from the per-scan poses."""
    p = mod.ReferencePipeline(**_kw(cfg))
    probe = mod.has_probe()
    run = dict(probe=probe, state=[], frames=[], weights=[], keyframes=[], cur=[], model_n=[], model_sha=[])
    for i, scan in enumerate(sequence(cfg[0])):
        p.compute(0.1 * i, scan)
        run["state"].append(p.state())
        if not probe:
            continue
        ids, w = p.frames()
        run["frames"].append(ids)
        run["weights"].append(w)
        run["keyframes"].append(p.keyframes())
        if leaves:
            run["cur"].append(p.current_leaves())
            m = p.model_leaves()
            run["model_n"].append(m.shape[0])
            run["model_sha"].append(_digest(m))
    traj = np.tile(np.eye(4), (len(run["state"]), 1, 1))
    traj[:, :3] = np.array(run["state"])[:, :12].reshape(-1, 3, 4)  # frame_to_map_ after each scan
    if probe:
        assert bits_equal(p.trajectory(), traj), _cid(cfg)
    run["traj"] = traj
    run["deskewed"] = {k: _deskew_shift(p, sequence(cfg[0])[k], run["traj"][k - 2:k]) for k in (2, 4)} if cfg[3] else None
    del p
    return run


def _deskew_shift(p, scan, prev):
    """How far the reference's deskew (pipeline.cpp:79-123) moves the points of a scan by the two poses before it.
    The deskewed cloud comes back sorted by azimuth: it is compared with the scan sorted the same way."""
    d = p.deskew(scan, prev[0], prev[1])
    order = np.argsort(np.arctan2(scan[:, 1], scan[:, 0]), kind="stable")
    return float(np.linalg.norm(d - scan[order], axis=1).max())


def _velocity_chis(run):
    """Every error norm chi of the velocity rounds (vel_estimator.cpp:45-79), recomputed from the run's trajectory and
    the velocity each round started from."""
    traj, st, ts = run["traj"], run["state"], 1.0 / HZ
    chis = []
    for i in range(1, len(traj)):
        odom = traj[max(0, i + 1 - FRAME_WINDOW): i + 1]
        X = st[i - 1][17:23]
        for j in range(len(odom) - 1):
            dt = (len(odom) - 1 - j) * ts
            T = np.linalg.inv(odom[j]) @ odom[-1]
            ang = [np.arctan2(-T[1, 2], T[2, 2]), np.arcsin(T[0, 2]), np.arctan2(-T[0, 1], T[0, 0])]
            e = np.concatenate([dt * X[:3] - T[:3, 3], dt * X[3:] - ang])
            chis.append(float(np.linalg.norm(e)))
    return np.array(chis)


def assert_coverage(run, cfg):
    """The run reached what its configuration is there for."""
    _, _, K, deskew, pth = cfg
    st = np.array(run["state"])
    n = st.shape[0]
    promoted = st[1:, 12].astype(bool)
    kf_before = np.concatenate([[1], st[:-1, 15]])[1:]
    evictions = int((promoted & (kf_before == K)).sum())
    probe = run["probe"]  # (the frames window, the keyframes and the inlier ratio need the probe)
    if pth == 0.0:  # never a promotion: the frames window rolls past FRAME_WINDOW
        assert not promoted.any() and (st[:, 15] == 1).all() and n - 1 > FRAME_WINDOW, _cid(cfg)
        ids = run["frames"][-1] if probe else range(n - FRAME_WINDOW, n)
        assert list(ids) == list(range(n - FRAME_WINDOW, n)), (_cid(cfg), ids)
    elif not promoted.any():  # a p_th the sequence never falls below: the window rolls over as well
        ids = run["frames"][-1] if probe else range(n - FRAME_WINDOW, n)
        assert _kw(cfg)["p_th"] < 0.8 and list(ids) == list(range(n - FRAME_WINDOW, n)), _cid(cfg)
    else:
        if pth == 1.0:  # a promotion on every scan that moved (a replayed scan matches every leaf of itself)
            assert promoted[2:14].all(), _cid(cfg)
        if K == 1 or pth == 1.0:
            assert evictions >= 1 and st[-1, 15] == K, (_cid(cfg), evictions)
    if probe:
        assert (promoted == (st[1:, 16] < _kw(cfg)["p_th"])).all(), _cid(cfg)
    if cfg[0] == "turns" and not deskew:  # the replayed sweeps at rest: frames 1 and 2 weigh the same, bit for bit
        assert bits_equal(st[1, :12], st[2, :12]), _cid(cfg)  # (registered to the same pose)
        if probe:
            ids, w = run["frames"][2], run["weights"][2]
            assert list(ids) == [1, 2] and w[0] == w[1] and st[1, 16] == st[2, 16] == 1.0, (_cid(cfg), w)
        if cfg[1] == "default" and pth != 0.0:  # and the first keyframe chosen after them is the first of the two
            first = int(np.argmax(promoted)) + 1
            assert first > 2 and st[first, 14] == 1, (_cid(cfg), first, st[first, 14])
    kfs = run["keyframes"] if probe else []
    assert all(len(k) == s[15] for k, s in zip(kfs, st)) and all(list(k) == sorted(k) for k in kfs), _cid(cfg)
    # the Huber scale of the velocity estimator is applied, clearly above its threshold
    chis = _velocity_chis(run)
    assert chis.max() > 1.5 * E_THRESHOLD_VEL, (_cid(cfg), chis.max())
    assert (chis < E_THRESHOLD_VEL).any(), _cid(cfg)
    if cfg[0] == "bumps":  # every velocity component moves
        assert (np.abs(st[:, 17:23]).max(axis=0) > 0.05).all(), (_cid(cfg), np.abs(st[:, 17:23]).max(axis=0))
    if cfg[0] == "turns":  # the standstill: the velocity decays towards zero
        speed = np.linalg.norm(st[:, 17:20], axis=1)
        assert speed.max() > 5.0 and speed[-1] < 0.2 * speed.max(), (_cid(cfg), speed)
    if deskew:  # deskewed from the third compute on (trajectory_.size() > 1), as soon as the vehicle moves
        k = 2 if cfg[0] == "bumps" else 4  # (turns: at rest up to scan 2)
        assert run["deskewed"][k] > 0.01, (_cid(cfg), run["deskewed"])


# ------------------------------------------------------------------ CPU: the probe, and coverage on the CPU reference
@pytest.fixture(scope="module")
def cpu_ref(built):
    from oracle import reference as R
    if not R.available():
        pytest.skip("the reference is not built (its sources are not present: oracle/reference.py REF_SRC)")
    R.lib()
    return R


@pytest.fixture(scope="module")
def cpu_probe(cpu_ref):
    if not cpu_ref.has_probe():
        pytest.skip("oracle/_ref/libmadicp_ref.so predates the Pipeline probe and the reference sources are not here to "
                    "rebuild it (oracle/reference.py REF_SRC)")
    return cpu_ref


def test_probe_inlier_ratio_equals_the_oracle_pipeline(cpu_probe, oracle):
    """The probe's inlier ratio (pipeline.cpp:197-204, recounted from the leaves' flags) == the oracle pipeline's
    st[16], bit for bit, scan after scan; NaN before the first registration."""
    cfg = ("turns", "default", 4, 0, None)
    ref, orc = cpu_probe.ReferencePipeline(**_kw(cfg)), oracle.OraclePipeline(**_kw(cfg))
    seen = set()
    for i, scan in enumerate(sequence("turns")[:12]):
        ref.compute(0.1 * i, scan)
        orc.compute(0.1 * i, scan)
        a, b = ref.state(), orc.state()
        if i == 0:
            assert np.isnan(a[16])
            continue
        assert bits_equal(a[16:17], b[16:17]), (i, a[16], b[16])
        assert (a[12:16] == b[12:16]).all(), i
        seen.add(a[16])
    assert len(seen) > 3 and 0.0 < min(seen) < 0.9 and max(seen) == 1.0  # (1.0: a replayed sweep)


def test_probe_lists_follow_the_pipeline(cpu_probe):
    """frames window, keyframes, leaves and trajectory of the probe are consistent with state()."""
    cfg = ("turns", "default", 4, 0, None)
    p = cpu_probe.ReferencePipeline(**_kw(cfg))
    assert p.frames()[0].size == 0 and p.keyframes().size == 0 and p.trajectory().shape == (0, 4, 4)
    for i, scan in enumerate(sequence("turns")[:6]):
        p.compute(0.1 * i, scan)
        st, traj = p.state(), p.trajectory()
        assert traj.shape == (i + 1, 4, 4) and bits_equal(traj[-1][:3], st[:12].reshape(3, 4))
        assert p.keyframes().size == st[15] and p.keyframes()[-1] == st[14]
        ids, w = p.frames()
        assert (np.diff(ids) > 0).all() and np.isfinite(w).all() and (ids > st[14]).all() if i else ids.size == 0
        cur, model = p.current_leaves(), p.model_leaves()
        assert (cur.shape[0] > 100) if i else (cur.shape[0] == 0)
        assert model.shape[0] > 100 and model.shape[1] == 3


CPU_COVERAGE = [("turns", "default", 1, 0, None), ("turns", "default", 4, 0, 1.0), ("turns", "default", 4, 0, 0.0),
                ("bumps", "default", 4, 1, None)]


@pytest.mark.parametrize("cfg", CPU_COVERAGE, ids=_cid)
def test_sequences_reach_their_branches_on_the_cpu_reference(cpu_ref, cfg):
    assert_coverage(reference_run(cpu_ref, cfg, leaves=False), cfg)


# ------------------------------------------------------------------ GPU 1: chained rounds == one-round launches
def _kf_case(K):
    """K keyframes spread over 12 m of the lane and a query 0.8 m past the last; the start is 0.5 m / 0.03 rad off."""
    beams, azimuths = (16, 512) if K == 64 else (32, 1024)
    scene = synth.StreetScene(seed=7)
    step = 12.0 / K
    base = [synth.pose_xyyaw(step * k, 1.0 + 0.2 * np.sin(0.3 * k), 0.01 * np.sin(0.2 * k)) for k in range(K)]
    trees = []
    for k, T in enumerate(base):
        ft = FlatTree(synth.lidar_scan(scene, T, beams=beams, azimuths=azimuths, seed=300 + k))
        ft.apply_transform(synth.sensor_pose(T))
        trees.append(ft)
    q = base[-1] @ synth.pose_xyyaw(0.8, 0.0, 0.02)
    query = synth.lidar_scan(scene, q, beams=beams, azimuths=azimuths, seed=299)
    X0 = synth.sensor_pose(q) @ synth.pose_xyyaw(0.5, -0.2, 0.03)
    reg = Registrar(device=0, max_keyframes=K)
    for k, ft in enumerate(trees):
        reg.put_keyframe(k, ft)
    reg.set_moving(FlatTree(query).leaf_means())
    return dict(reg=reg, trees=trees, X0=X0)


@pytest.fixture(scope="module")
def kf_cases():
    cache = {}

    def get(K):
        if K not in cache:
            cache[K] = _kf_case(K)
        return cache[K]
    return get


def _one_round_chain(reg, X0, n):
    """n launches of one round, each from the previous one's pose: poses X[0..n], and each launch's outputs."""
    X, outs = [np.asarray(X0, dtype=np.float64)[:3].copy()], []
    for _ in range(n):
        o = reg.register(X[-1], 1)
        X.append(o["X"])
        outs.append(o)
    return np.array(X), outs


def _fetch_weight(reg, X0, n, partial=False):
    reg.register_async(X0, n, partial=partial)
    return reg.register_fetch(want_matched=True)


@pytest.mark.gpu
@pytest.mark.parametrize("pname", list(PARAMS))
@pytest.mark.parametrize("K", [1, 4, 16, 64])
def test_chained_rounds_equal_one_round_launches(kf_cases, K, pname):
    """register(X0, n) == n calls of register(X, 1), each from the previous call's pose: every round's pose, the last
    round's H/b and flags, and the keyframe weight -- in every memo mode, for n = 15 (one launch) and n = 70 (a 64-round
    launch chained to a 6-round one)."""
    case = kf_cases(K)
    reg, X0 = case["reg"], case["X0"]
    reg.set_params(*PARAMS[pname])
    try:
        for mode in (0, 1, 2):
            reg.set_memo(mode)
            for n in (15, 70):
                what = (K, pname, mode, n)
                X, outs = _one_round_chain(reg, X0, n)
                full = reg.register(X0, n)
                tr = reg.register_trace()
                start = ((n - 1) // MAX_ITERS) * MAX_ITERS  # the trace is the last launch's
                assert bits_equal(tr, X[start:]), (what, "trace", _first_row(tr, X[start:]))
                assert bits_equal(full["X"], X[n]), what
                for k in ("H", "b"):
                    assert bits_equal(full[k], outs[-1][k]), (what, k)
                assert (full["matched"] == outs[-1]["matched"]).all() and full["n_matched"] == outs[-1]["n_matched"], what
                one = _fetch_weight(reg, X[n - 1], 1)
                if n <= MAX_ITERS:
                    f = _fetch_weight(reg, X0, n)
                    for k in ("X", "H", "b"):
                        assert bits_equal(f[k], full[k]), (what, "fetch", k)
                    assert bits_equal(f["weight"], one["weight"]), (what, "weight", f["weight"], one["weight"])
                else:
                    reg.register(X0, MAX_ITERS)
                    assert bits_equal(reg.register_trace(), X[:MAX_ITERS + 1]), (what, "first launch")
                    assert bits_equal(reg.inv_det6(full["H"]), one["weight"]), (what, "weight")
                assert outs[0]["n_matched"] > 0 and not bits_equal(X[1], X[0]), what
    finally:
        reg.set_memo(2)
        reg.set_params(*PARAMS["default"])


def _first_row(a, b):
    if a.shape != b.shape:
        return ("shape", a.shape, b.shape)
    bad = [i for i in range(a.shape[0]) if not bits_equal(a[i], b[i])]
    return ("first round apart", bad[0] if bad else None)


@pytest.mark.gpu
def test_partial_flags_are_the_union_of_one_round_launches(kf_cases):
    case = kf_cases(4)
    reg, X0 = case["reg"], case["X0"]
    X, outs = _one_round_chain(reg, X0, 7)
    f = _fetch_weight(reg, X0, 7, partial=True)
    union = np.zeros_like(outs[0]["matched"], dtype=bool)
    for o in outs:
        union |= o["matched"].astype(bool)
    assert bits_equal(f["X"], X[7]) and bits_equal(f["H"], outs[-1]["H"]) and bits_equal(f["b"], outs[-1]["b"])
    assert (f["matched"].astype(bool) == union).all() and f["n_matched"] == int(union.sum())
    assert (union & ~outs[-1]["matched"].astype(bool)).any()  # the earlier rounds do add flags here


# ------------------------------------------------------------------ GPU 2: Pipeline == the reference over the backend
@pytest.fixture(scope="module")
def ref_gpu(built):
    from oracle import reference as R
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmadicp_ref_gpu.so")) and not os.path.isdir(R.REF_SRC):
        pytest.skip("oracle/_ref/libmadicp_ref_gpu.so not built (it needs the reference sources, oracle/reference.py REF_SRC)")
    G = R.variant("libmadicp_ref_gpu.so", "ref_gpu")
    G.lib()
    return G


@pytest.fixture(scope="module")
def ref_runs(ref_gpu):
    """The reference's run of each configuration, computed once."""
    cache = {}

    def get(cfg):
        if cfg not in cache:
            cache[cfg] = reference_run(ref_gpu, cfg)
            gc.collect()
            ref_gpu.lib().madicp_b200_backend_release_all()  # (its MADicp has no destructor to free the context)
        return cache[cfg]
    return get


ROUTES = ["compute", "lookahead", "host", "keep_map"]


def run_pipeline(cfg, route, ref, depth=5):
    """cfg's sequence through Pipeline by `route`, held after every scan to the reference's run."""
    from mad_icp_b200.pybind.pypeline import Pipeline
    extra = dict(keep_cloud=True, map_voxel_size=0.5) if route == "keep_map" else {}
    with mock.patch.dict(os.environ, {"MADICP_GPU_BUILD": "0" if route == "host" else "1"}):
        p = Pipeline(**_kw(cfg), **extra)
    scans = sequence(cfg[0])
    n, queued = len(scans), 0
    depth = depth if route == "lookahead" else 0
    for i, scan in enumerate(scans):
        while depth and queued < min(i + depth, n):
            assert p.prefetch(scans[queued], deskew_ahead=bool(cfg[3]))
            queued += 1
        p.compute(0.1 * i, scan)
        queued = max(queued, i + 1)
        st, where = ref["state"][i], (_cid(cfg), route, "scan", i)
        pose = p.currentPose()
        assert bits_equal(pose[:3], st[:12].reshape(3, 4)), (where, "pose", np.abs(pose[:3] - st[:12].reshape(3, 4)).max())
        assert (p.isMapUpdated(), p.currentID(), p.keyframeID(), p.numKeyframes()) == \
            (bool(st[12]), int(st[13]), int(st[14]), int(st[15])), (where, "keyframe decision", st[12:16])
        assert bits_equal(p.keyframePose(), ref["traj"][int(st[14])]), (where, "keyframe pose")
        if not ref["probe"]:  # (a reference library without the probe: no inlier ratio, no leaves)
            continue
        model = p.modelLeavesArray()
        assert model.shape[0] == ref["model_n"][i] and _digest(model) == ref["model_sha"][i], (where, "model leaves")
        if i == 0:  # the reference hands out no current leaves before its first registration (see the module doc)
            continue
        assert bits_equal(p.inliersRatio(), st[16]), (where, "inlier ratio", p.inliersRatio(), st[16])
        assert bits_equal(p.currentLeavesArray(), ref["cur"][i]), (where, "current leaves")
    traj = np.array(p.trajectory())
    assert traj.shape == ref["traj"].shape and bits_equal(traj, ref["traj"]), (_cid(cfg), route, "trajectory")
    if route == "keep_map":
        assert p.mapSize() > 0
    if route == "lookahead" and not cfg[3]:
        assert p.prefetched() == 0


@pytest.mark.gpu
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cid)
def test_reference_run_reaches_its_branches(ref_runs, cfg):
    assert_coverage(ref_runs(cfg), cfg)


@pytest.mark.gpu
@pytest.mark.parametrize("route", ROUTES)
@pytest.mark.parametrize("cfg", CONFIGS, ids=_cid)
def test_pipeline_equals_the_reference_pipeline(ref_runs, cfg, route):
    run_pipeline(cfg, route, ref_runs(cfg))


@pytest.mark.gpu
def test_pipeline_equals_the_reference_pipeline_at_the_bench_shape(ref_runs):
    """100 sweeps of 64 x 2048, 16 keyframes, look-ahead: the configuration bench.py times."""
    ref = ref_runs(BIG)
    st = np.array(ref["state"])
    assert st[1:, 12].sum() >= 5  # the model grows
    run_pipeline(BIG, "lookahead", ref, depth=8)


# ------------------------------------------------------------------ GPU 3: MADicp.compute == the backend's loop
@pytest.mark.gpu
@pytest.mark.parametrize("pname", list(PARAMS))
def test_madicp_compute_equals_the_backend_loop(ref_gpu, pname):
    """pymadicp's MADicp.compute (one launch of all rounds) == the reference's registration loop over the backend
    (one launch per round), bit for bit, at 15 rounds and at 1."""
    from mad_icp_b200.pybind.pymadicp import MADicp
    min_ball, rho_ker, b_ratio = PARAMS[pname]
    c = synth.registration_case(K=1, beams=32, azimuths=1024, seed=11)
    ref_cloud, query = c["scans"][0], c["query"]
    T0 = np.linalg.inv(c["kf_poses"][0]) @ c["T_guess"]
    m = MADicp(num_threads=4)
    m.setReferenceCloud(ref_cloud, b_max=min_ball, b_min=0.1 if min_ball > 0.1 else 0.05)
    m.setQueryCloud(query, b_max=min_ball, b_min=0.1 if min_ball > 0.1 else 0.05)
    kf = ref_gpu.ReferenceTree(ref_cloud, b_max=min_ball, b_min=0.1 if min_ball > 0.1 else 0.05)
    mv = ref_gpu.ReferenceTree(query, b_max=min_ball, b_min=0.1 if min_ball > 0.1 else 0.05)
    for iters in (15, 1):
        want = ref_gpu.icp_run([kf], mv, T0, iters=iters, min_ball=min_ball, rho_ker=rho_ker, b_ratio=b_ratio,
                               num_threads=4)
        got = m.compute(T0, icp_iterations=iters, rho_ker=rho_ker, b_ratio=b_ratio)
        assert bits_equal(got[:3], want["X"]), (pname, iters, np.abs(got[:3] - want["X"]).max())
    del kf, mv
    gc.collect()
    ref_gpu.lib().madicp_b200_backend_release_all()
