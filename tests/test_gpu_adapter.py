"""The drop-in boundary, proven (`-m gpu`): oracle/_ref/libmadicp_ref_gpu.so is the reference's UNMODIFIED
odometry/pipeline.cpp + odometry/vel_estimator.cpp, compiled against its own headers and linked with
mad_icp_b200/csrc/adapter/reference_backend.cpp in place of its tools/mad_tree.cpp + odometry/mad_icp.cpp
(`make -C oracle ref_gpu`, run by build() where the reference's sources are: oracle/reference.py REF_SRC).  It is driven through the same C
entry points (oracle/ref_capi.cpp) as the CPU build of the reference, and must agree with it: keyframe decisions
equal scan for scan, poses within 1e-5 rad / 1e-4 m, registration loop H/b 1e-12, correspondences bit-exact."""
import os

import numpy as np
import pytest

from mad_icp_b200 import synth
from util import HB_REL, POSE_M, POSE_RAD, pose_error

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def libs():
    from oracle import reference as R
    if not os.path.exists(os.path.join(ROOT, "oracle", "_ref", "libmadicp_ref_gpu.so")) and not os.path.isdir(R.REF_SRC):
        pytest.skip("oracle/_ref/libmadicp_ref_gpu.so not built (it needs the reference sources, oracle/reference.py REF_SRC)")
    G = R.variant("libmadicp_ref_gpu.so", "ref_gpu")
    R.lib()
    G.lib()
    return R, G


def test_unmodified_pipeline_over_the_gpu_backend_streams_like_the_cpu_reference(libs):
    R, G = libs
    seq = synth.sequence(n_scans=24, beams=32, azimuths=1024, seed=4)
    kw = dict(sensor_hz=10.0, deskew=False, b_max=0.2, rho_ker=0.1, p_th=0.8, b_min=0.1, b_ratio=0.02, num_keyframes=4,
              num_threads=4, realtime=False)
    pc, pg = R.ReferencePipeline(**kw), G.ReferencePipeline(**kw)
    promoted = 0
    for i, scan in enumerate(seq["scans"]):
        pc.compute(0.1 * i, scan)
        pg.compute(0.1 * i, scan)
        sc, sg = pc.state(), pg.state()
        assert (sc[12:16] == sg[12:16]).all(), f"scan {i}: keyframe decision differs {sc[12:16]} vs {sg[12:16]}"
        ang, dt = pose_error(sc[:12].reshape(3, 4), sg[:12].reshape(3, 4))
        assert ang < POSE_RAD and dt < POSE_M, (i, ang, dt)
        assert np.abs(sc[17:23] - sg[17:23]).max() < 1e-6
        promoted += int(sc[12])
    assert promoted >= 3, "the sequence must exercise keyframe promotion and eviction"


def test_deskewed_stream(libs):
    """With deskew the previous pose ESTIMATES (equal to ~1e-12 between the two builds, not bit-equal) are applied to
    the cloud before the tree is built, and the build is discontinuous in its input -- the synthetic walls put many
    points exactly on split planes -- so the two runs register slightly different leaf sets and agree at the
    sensor-noise level (the same bar as tests/test_pybind_api.py uses for the facade's Pipeline)."""
    R, G = libs
    seq = synth.sequence(n_scans=8, beams=16, azimuths=512, seed=6)
    kw = dict(sensor_hz=10.0, deskew=True, num_keyframes=2, num_threads=2)
    pc, pg = R.ReferencePipeline(**kw), G.ReferencePipeline(**kw)
    for i, scan in enumerate(seq["scans"]):
        pc.compute(0.1 * i, scan)
        pg.compute(0.1 * i, scan)
        sc, sg = pc.state(), pg.state()
        assert sc[13] == sg[13], i
        ang, dt = pose_error(sc[:12].reshape(3, 4), sg[:12].reshape(3, 4))
        assert ang < 5e-3 and dt < 5e-2, (i, ang, dt)
        if i < 2:  # not deskewed yet (pipeline.cpp:137): lock-step
            assert ang < POSE_RAD and dt < POSE_M and (sc[12:16] == sg[12:16]).all(), i


def test_reference_madicp_calls_on_the_gpu(libs):
    """MADicp::setMoving / init / resetAdders / update (under OpenMP) / updateState of the reference's class, backed by
    the GPU: every round's pose and H/b against the CPU build, matched flags, trees identical node for node."""
    R, G = libs
    case = synth.registration_case(K=3, beams=16, azimuths=512, seed=2)
    kc, kg = [], []
    for s, P in zip(case["scans"], case["kf_poses"]):
        a, b = R.ReferenceTree(s), G.ReferenceTree(s)
        ea, eb = a.export(), b.export()
        for k in ea:
            assert np.array_equal(ea[k], eb[k], equal_nan=True), k  # the backend's MADtree IS the reference's tree
        a.apply_transform(P)
        b.apply_transform(P)
        assert np.array_equal(a.export()["mean"], b.export()["mean"])
        kc.append(a)
        kg.append(b)
    mc, mg = R.ReferenceTree(case["query"]), G.ReferenceTree(case["query"])
    rc = R.icp_run(kc, mc, case["T_guess"], iters=10, num_threads=3, record_idx=True)
    rg = G.icp_run(kg, mg, case["T_guess"], iters=10, num_threads=3, record_idx=True)
    assert (rc["idx_hist"][0] == rg["idx_hist"][0]).all()  # same pose in round 0 -> identical correspondences
    for it in range(10):
        ang, dt = pose_error(rc["X_hist"][it], rg["X_hist"][it])
        assert ang < 1e-9 and dt < 1e-9, it
        scale = np.abs(rc["H_hist"][it]).max()
        assert np.abs(rc["H_hist"][it] - rg["H_hist"][it]).max() / scale < 100 * HB_REL
    ang, dt = pose_error(rc["X"], rg["X"])
    assert ang < POSE_RAD and dt < POSE_M
    assert (rc["matched"] == rg["matched"]).all()
