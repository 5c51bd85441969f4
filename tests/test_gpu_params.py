"""Registration at other ICP parameters than the defaults, and across set_params on a live context (`-m gpu`).

min_ball, rho_ker and b_ratio reach every kernel on the hot path: the gate radius min_ball + b_ratio*|p|
(k_prepare_moving, the gate of linearize_one, the checkpoint depth of round 0), sqrt(rho_ker) (the Huber threshold) and
the planarity weight (1 - bbox0/min_ball)^2, held twice -- in the leaf codes of the quad records, read by the items that
walk, and in the per-node ww table, read by the items whose walk the path memo skips.  madicp_set_params re-runs
prepare_slot on every resident slot when min_ball changes and marks the gate radii stale otherwise.

The oracle's ICP loop is pinned to the reference's own sources at the SWEEP sets (tests/test_reference_pin.py), so
the comparisons against it below reach the reference transitively.  Bars as in tests/test_gpu_parity.py: indices and
flags exact, H/b HB_REL, pose POSE_RAD / POSE_M."""
import math
import os

import numpy as np
import pytest

from mad_icp_b200 import FlatTree, MadIcpError, Registrar, synth
from test_pybind_api import _sequence
from test_reference_pin import SWEEP
from util import HB_REL, POSE_M, POSE_RAD, bits_equal, pose_error

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

DEFAULT = (0.2, 0.1, 0.02)  # (min_ball, rho_ker, b_ratio)
# (b_max, b_min) of the trees, then (min_ball, rho_ker, b_ratio)
_SETS = [((b_max, b_min), (b_max, rho_ker, b_ratio)) for b_max, b_min, rho_ker, b_ratio in SWEEP] + [
    ((0.2, 0.1), (0.2, 0.0, 0.02)),        # rho_ker = 0: Huber scale 0 for every nonzero residual
    ((0.2, 0.1), (0.2, math.inf, 0.02)),   # no Huber
    ((0.2, 0.1), (0.2, 0.1, 1e3)),         # every pair inside the gate
    ((0.2, 0.1), (0.05, 0.1, 0.02)),       # min_ball < the trees' b_max: w < 0, weights above 1
    ((0.2, 0.1), (0.2, 0.1, -0.05)),       # negative gate radius: every pair rejected, as `norm > ball` does
    ((0.2, 0.1), (0.2, 0.1, math.nan)),    # NaN gate radius: every pair accepted, as `norm > NaN` is false
]
SETS = list(dict.fromkeys(_SETS, None))  # SWEEP may hold some of the others
SET_IDS = ["tree%g-%g_P%g-%g-%g" % (t + p) for t, p in SETS]

CASE = dict(K=2, beams=16, azimuths=512, seed=9)  # the case of test_reference_pin.case_parameter_sweep
_cases = {}


def _case(O, b_max=0.2, b_min=0.1):
    """The case's keyframe trees (host-built, in the map frame) and moving tree, GPU and oracle side, cached."""
    key = (b_max, b_min)
    if key not in _cases:
        c = synth.registration_case(**CASE)
        fts, ots = [], []
        for scan, P in zip(c["scans"], c["kf_poses"]):
            ft, ot = FlatTree(scan, b_max=b_max, b_min=b_min), O.OracleTree(scan, b_max=b_max, b_min=b_min)
            ft.apply_transform(P)
            ot.apply_transform(P)
            fts.append(ft)
            ots.append(ot)
        fq = FlatTree(c["query"], b_max=b_max, b_min=b_min)
        _cases[key] = dict(c=c, fts=fts, ots=ots, fq=fq, means=fq.leaf_means(),
                           oq=O.OracleTree(c["query"], b_max=b_max, b_min=b_min))
    return _cases[key]


def _registrar(cs, params=DEFAULT, slots=None, moving="means"):
    reg = Registrar(device=0, max_keyframes=len(cs["fts"]), min_ball=params[0], rho_ker=params[1], b_ratio=params[2])
    for k in (range(len(cs["fts"])) if slots is None else slots):
        reg.put_keyframe(k, cs["fts"][k])
    _set_moving(reg, cs, moving)
    return reg


def _set_moving(reg, cs, moving):
    if moving == "means":
        reg.set_moving(cs["means"])
    else:  # the scan's tree built on this context's device, its leaves straight to the kernel
        reg._moving_tree = reg.build_tree(cs["c"]["query"], b_max=cs["fq"].b_max, b_min=cs["fq"].b_min)
        reg.set_moving_tree(reg._moving_tree)


def _run(reg, X0, iters=10):
    r = reg.register(X0, iters=iters)
    r["trace"] = reg.register_trace()
    return r


def _assert_bits(a, b, what):
    for k in ("X", "H", "b", "trace"):
        assert bits_equal(a[k], b[k]), (what, k)
    assert (a["matched"] == b["matched"]).all() and a["n_matched"] == b["n_matched"], what


def _check_Hb(H, b, H_ref, b_ref):
    scale = max(np.abs(H_ref).max(), np.abs(b_ref).max())
    if scale == 0:  # nothing the oracle accepted contributed
        assert not H.any() and not b.any(), (np.abs(H).max(), np.abs(b).max())
        return
    eh, eb = float(np.abs(H - H_ref).max() / scale), float(np.abs(b - b_ref).max() / scale)
    assert eh <= HB_REL and eb <= HB_REL, (eh, eb)


# ------------------------------------------------------------------ 1. oracle parity per parameter set
@pytest.mark.parametrize("trees,P", SETS, ids=SET_IDS)
def test_parity_with_the_oracle(oracle, trees, P):
    cs = _case(oracle, *trees)
    c, kw = cs["c"], dict(zip(("min_ball", "rho_ker", "b_ratio"), P))
    reg = _registrar(cs, P)
    ref = oracle.icp_run(cs["ots"], cs["oq"], c["T_guess"], iters=10, num_threads=2, **kw)
    out = reg.register(c["T_guess"], iters=10)
    if P[2] < 0:  # every gate radius of the case is negative (|mean| > 4 m): nothing matches, the pose stays
        assert out["n_matched"] == 0, f"a negative gate radius matched {out['n_matched']} moving leaves"
        assert not out["H"].any() and not out["b"].any()
        assert bits_equal(out["X"], c["T_guess"][:3])
    ang, dt = pose_error(out["X"], ref["X"])
    assert ang < POSE_RAD and dt < POSE_M, (ang, dt)
    assert (out["matched"] == ref["matched"]).all(), (out["n_matched"], int(ref["matched"].sum()))
    for it in range(10):
        X = ref["X_hist"][it]
        idx = reg.search(X)
        assert (idx == ref["idx_hist"][it]).all(), f"round {it}: {int((idx != ref['idx_hist'][it]).sum())} indices differ"
        H, b, m = reg.linearize(X)
        Ho, bo, mo = oracle.icp_linearize(cs["ots"], cs["oq"], X, **kw)
        assert (m == mo).all(), f"round {it}: {int((m != mo).sum())} flags differ, gpu {int(m.sum())} oracle {int(mo.sum())}"
        _check_Hb(H, b, Ho, bo)
    # the same loop driven from the host through the step API
    X = np.array(c["T_guess"][:3], dtype=np.float64)
    for _ in range(10):
        H, b, m = reg.linearize(X)
        X = reg.solve_update(H, b, X)
    ang, dt = pose_error(out["X"], X)
    assert ang < 1e-9 and dt < 1e-9, (ang, dt)
    assert (m == out["matched"]).all()
    if math.isnan(P[2]):
        assert out["matched"].all()


# ------------------------------------------------------------------ 2. set_params on a live context == a fresh one
GATE_ONLY = (0.2, 0.3, 0.05)   # same min_ball: the gate radii are rebuilt at the next launch (mov4_stale)
REWEIGH = (0.1, 0.05, 0.01)    # another min_ball: prepare_slot re-runs on every resident slot


@pytest.mark.parametrize("moving", ["means", "tree"])
@pytest.mark.parametrize("late_keyframes", [False, True], ids=["kf_before", "kf_after"])
@pytest.mark.parametrize("P", [GATE_ONLY, REWEIGH], ids=["gate_only", "reweigh"])
def test_set_params_on_a_live_context_equals_a_fresh_one(oracle, P, late_keyframes, moving):
    cs = _case(oracle)
    X0 = cs["c"]["T_guess"]
    K = len(cs["fts"])
    live = _registrar(cs, DEFAULT, slots=[0] if late_keyframes else None, moving=moving)
    first = _run(live, X0)
    live.set_params(*P)
    if late_keyframes:
        for k in range(1, K):
            live.put_keyframe(k, cs["fts"][k])
    got = _run(live, X0)
    fresh = _registrar(cs, P, moving=moving)
    _assert_bits(got, _run(fresh, X0), "live vs fresh")
    live.set_params(*DEFAULT)
    if late_keyframes:
        for k in range(1, K):
            live.drop_keyframe(k)
    _assert_bits(_run(live, X0), first, "back to the defaults")


def test_set_params_between_register_async_and_fetch(oracle):
    """The launch in flight keeps the parameters it was enqueued with; the next one uses the new ones."""
    cs = _case(oracle)
    X0 = cs["c"]["T_guess"]
    want_old = _run(_registrar(cs, DEFAULT), X0)
    want_new = _run(_registrar(cs, REWEIGH), X0)
    for P, want in ((REWEIGH, want_new), (GATE_ONLY, _run(_registrar(cs, GATE_ONLY), X0))):
        live = _registrar(cs, DEFAULT)
        live.register_async(X0, 10)
        live.set_params(*P)
        old = live.register_fetch(want_matched=True)
        old["trace"] = live.register_trace()
        _assert_bits(old, want_old, ("fetch after set_params", P))
        _assert_bits(_run(live, X0), want, ("next register", P))
    assert not bits_equal(want_old["H"], want_new["H"])  # the two sets do differ


# ------------------------------------------------------------------ 3. both copies of the planarity weight
def _memo_modes(reg, X0):
    out = []
    for mode in (0, 1, 2):
        reg.set_memo(mode)
        out.append(_run(reg, X0))
    reg.set_memo(True)
    return out


@pytest.mark.parametrize("trees,P", SETS, ids=SET_IDS)
def test_memo_modes_agree_after_set_params(oracle, trees, P):
    """Mode 0 reads the weight from the quad records' leaf codes only; modes 1 and 2 read the ww table for the items
    whose walk they skip.  After set_params (a reweigh wherever min_ball differs from the default) all three must give
    the same bits, from the guess and from 1.5 m off it; the gate radius is also round 0's checkpoint depth."""
    cs = _case(oracle, *trees)
    reg = _registrar(cs, DEFAULT)
    _run(reg, cs["c"]["T_guess"])
    reg.set_params(*P)
    for shift in (0.0, 1.5):
        X0 = np.array(cs["c"]["T_guess"], dtype=np.float64)
        X0[0, 3] += shift
        runs = _memo_modes(reg, X0)
        for mode, r in enumerate(runs[1:], start=1):
            _assert_bits(r, runs[0], (shift, mode))


# ------------------------------------------------------------------ 4. the gate at its boundary
def test_gate_boundary_to_the_ulp(oracle):
    """b_ratio = 0, so the gate radius is min_ball exactly.  For ~20 (moving leaf, fixed leaf) pairs the distance is
    computed with the reference's arithmetic (ml = X*m row by row without FMA, the difference, (a0^2 + a1^2) + a2^2,
    sqrt), min_ball is set to it and to its neighbours 1 and 2 ulp away: the pair is matched at and above its
    distance, not below -- d^2 lies in the 1e-14 band there, so linearize_one decides through its sqrt."""
    cs = _case(oracle)
    c = cs["c"]
    X = np.array(c["T_guess"][:3], dtype=np.float64)
    reg = Registrar(device=0, max_keyframes=1, min_ball=0.2, rho_ker=0.1, b_ratio=0.0)
    reg.put_keyframe(0, cs["fts"][0])
    reg.set_moving(cs["means"])
    ot = [cs["ots"][0]]
    fixed = cs["fts"][0].leaves()[0]
    assert bits_equal(fixed, cs["ots"][0].leaves()[0])
    m = cs["means"]
    f = fixed[reg.search(X)[0]]
    R, t = X[:, :3], X[:, 3]
    ml = ((R[:, 0] * m[:, :1] + R[:, 1] * m[:, 1:2]) + R[:, 2] * m[:, 2:3]) + t  # numpy: no FMA
    d = ml - f
    dist = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
    pool = np.flatnonzero((dist > 0.02) & (dist < 1.0))
    assert pool.size >= 20
    picks = np.random.RandomState(0).choice(pool, 20, replace=False)
    for q in picks:
        ball = dist[q]
        for step in (-2, -1, 0, 1, 2):
            mb = ball
            for _ in range(abs(step)):
                mb = np.nextafter(mb, np.inf if step > 0 else -np.inf)
            reg.set_params(float(mb), 0.1, 0.0)
            H, b, flags = reg.linearize(X)
            Ho, bo, fo = oracle.icp_linearize(ot, cs["oq"], X, min_ball=float(mb), rho_ker=0.1, b_ratio=0.0)
            assert bool(fo[q]) == (step >= 0), (q, step)  # the oracle's own arithmetic agrees with the numpy above
            assert (flags == fo).all(), (q, step, int((flags != fo).sum()))
            one = reg.register(X, iters=1)  # round 0 of the persistent kernel decides at the same pose
            assert (one["matched"] == fo).all(), (q, step)


# ------------------------------------------------------------------ 5. rejected arguments
BAD = [(0.0, 0.1, 0.02), (-1.0, 0.1, 0.02), (math.nan, 0.1, 0.02), (0.2, -1.0, 0.02)]


def test_rejected_set_params_leave_the_parameters_in_force(oracle):
    empty = Registrar(device=0, max_keyframes=1)
    for bad in BAD:
        with pytest.raises(MadIcpError, match="madicp_set_params: "):
            empty.set_params(*bad)
    cs = _case(oracle)
    X0 = cs["c"]["T_guess"]
    reg = _registrar(cs, REWEIGH)
    before = _run(reg, X0)
    for bad in BAD:
        with pytest.raises(MadIcpError, match="madicp_set_params: "):
            reg.set_params(*bad)
        _assert_bits(_run(reg, X0), before, bad)


# ------------------------------------------------------------------ 6. Pipeline at other parameters
PIPE_SETS = [(0.4, 0.2, 0.3, 0.95, 0.05), (0.1, 0.05, 0.05, 0.5, 0.01)]  # (b_max, b_min, rho_ker, p_th, b_ratio)


def test_pipeline_tracks_like_the_oracle_at_other_parameters(oracle):
    from mad_icp_b200.pybind.pypeline import Pipeline
    promotions = []
    for b_max, b_min, rho_ker, p_th, b_ratio in PIPE_SETS:
        kw = dict(sensor_hz=10.0, deskew=False, b_max=b_max, rho_ker=rho_ker, p_th=p_th, b_min=b_min, b_ratio=b_ratio,
                  num_keyframes=4, num_threads=4, realtime=False)
        ref, pipe = oracle.OraclePipeline(**kw), Pipeline(**kw)
        promoted = 0
        for i, (stamp, pts) in enumerate(_sequence(25)):
            ref.compute(stamp, pts)
            pipe.compute(stamp, pts)
            st = ref.state()
            ang, dt = pose_error(pipe.currentPose(), st[:12].reshape(3, 4))
            assert ang < POSE_RAD and dt < POSE_M, (b_max, i, ang, dt)
            assert pipe.currentID() == int(st[13]) and pipe.isMapUpdated() == bool(st[12]), (b_max, i)
            assert pipe.keyframeID() == int(st[14]) and pipe.numKeyframes() == int(st[15]), (b_max, i)
            promoted += int(st[12])
        promotions.append(promoted)
    assert max(promotions) >= 3, promotions


# ------------------------------------------------------------------ 7. pymadicp.MADicp
def test_pymadicp_compute_rebuilds_on_every_change(oracle):
    """The facade rebuilds its context when rho_ker, b_ratio or the reference cloud's b_max change; each result must
    be a fresh wrapper's with the same arguments, bit for bit, and the oracle's with min_ball = the reference's b_max."""
    from mad_icp_b200.pybind.pymadicp import MADicp
    c = synth.registration_case(K=1, beams=16, azimuths=512, seed=9)
    ref_pts, query = c["scans"][0], c["query"]
    T = np.linalg.inv(c["kf_poses"][0]) @ c["T_guess"]  # the guess in the keyframe's own frame
    # (reference b_max, b_min), (query b_max, b_min), rho_ker, b_ratio -- applied in this order to one wrapper
    steps = [((0.2, 0.1), (0.2, 0.1), 0.05, 0.01), ((0.2, 0.1), (0.2, 0.1), 0.3, 0.05),
             ((0.4, 0.2), (0.2, 0.1), 0.3, 0.05), ((0.4, 0.2), (0.1, 0.05), 0.3, 0.05)]
    live, have = MADicp(num_threads=1), (None, None)
    outs = []
    for rb, qb, rho_ker, b_ratio in steps:
        if rb != have[0]:
            live.setReferenceCloud(ref_pts, b_max=rb[0], b_min=rb[1])
        if qb != have[1]:
            live.setQueryCloud(query, b_max=qb[0], b_min=qb[1])
        have = (rb, qb)
        got = live.compute(T, icp_iterations=10, rho_ker=rho_ker, b_ratio=b_ratio)
        outs.append(got)
        fresh = MADicp(num_threads=1)
        fresh.setReferenceCloud(ref_pts, b_max=rb[0], b_min=rb[1])
        fresh.setQueryCloud(query, b_max=qb[0], b_min=qb[1])
        want = fresh.compute(T, icp_iterations=10, rho_ker=rho_ker, b_ratio=b_ratio)
        assert bits_equal(got, want), (rb, qb, rho_ker, b_ratio)
        r = oracle.icp_run([oracle.OracleTree(ref_pts, b_max=rb[0], b_min=rb[1])],
                           oracle.OracleTree(query, b_max=qb[0], b_min=qb[1]), T, iters=10, min_ball=rb[0],
                           rho_ker=rho_ker, b_ratio=b_ratio, record=False)
        ang, dt = pose_error(got, r["X"])
        assert ang < POSE_RAD and dt < POSE_M, (rb, qb, rho_ker, b_ratio, ang, dt)
    assert not bits_equal(outs[0], outs[1]) and not bits_equal(outs[1], outs[2])


# ------------------------------------------------------------------ 8. the reference's Pipeline over the GPU backend
def test_unmodified_reference_pipeline_over_the_gpu_backend_at_other_parameters():
    from oracle import reference as R
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmadicp_ref_gpu.so")) and not os.path.isdir(R.REF_SRC):
        pytest.skip("oracle/_ref/libmadicp_ref_gpu.so not built (it needs the reference sources, oracle/reference.py REF_SRC)")
    G = R.variant("libmadicp_ref_gpu.so", "ref_gpu")
    R.lib()
    G.lib()
    b_max, b_min, rho_ker, p_th, b_ratio = PIPE_SETS[0]
    kw = dict(sensor_hz=10.0, deskew=False, b_max=b_max, rho_ker=rho_ker, p_th=p_th, b_min=b_min, b_ratio=b_ratio,
              num_keyframes=4, num_threads=4, realtime=False)
    seq = synth.sequence(n_scans=24, beams=32, azimuths=1024, seed=4)
    pc, pg = R.ReferencePipeline(**kw), G.ReferencePipeline(**kw)
    promoted = 0
    for i, scan in enumerate(seq["scans"]):
        pc.compute(0.1 * i, scan)
        pg.compute(0.1 * i, scan)
        sc, sg = pc.state(), pg.state()
        assert (sc[12:16] == sg[12:16]).all(), f"scan {i}: keyframe decision differs {sc[12:16]} vs {sg[12:16]}"
        ang, dt = pose_error(sc[:12].reshape(3, 4), sg[:12].reshape(3, 4))
        assert ang < POSE_RAD and dt < POSE_M, (i, ang, dt)
        promoted += int(sc[12])
    assert promoted >= 3
