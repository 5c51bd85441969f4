"""Auto-enabled when a real Eigen is on disk (SURVEY H1 / DESIGN.md section 2): compiles the reference's own
sources against REAL Eigen and requires the restatement (oracle/) to agree with it bit for bit -- trees, every
GN round, correspondences -- and learns Eigen's 3-term dot-product order with a discriminating vector.
This image has no Eigen (the reference fetches 3.4.0 at configure time), so here the module skips; on a box
that has it (EIGEN3_INCLUDE_DIR, /usr/include/eigen3, /usr/local/include/eigen3, baseline/_ref/**/Eigen)
the oracle's last unpinned piece becomes pinned without a code change."""
import glob
import os
import subprocess

import numpy as np
import pytest

from mad_icp_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from oracle.reference import REF_SRC  # noqa: E402


def _find_eigen():
    cands = [os.environ.get("EIGEN3_INCLUDE_DIR"), "/usr/include/eigen3", "/usr/local/include/eigen3", "/usr/include",
             "/usr/local/include"]
    cands += [os.path.dirname(os.path.dirname(p)) for p in
              glob.glob(os.path.join(ROOT, "baseline", "_ref", "**", "Eigen", "Core"), recursive=True)]
    for c in cands:
        if c and os.path.isfile(os.path.join(c, "Eigen", "Core")) and "eigen_standin" not in c:
            return c
    return None


EIGEN = _find_eigen()
pytestmark = pytest.mark.skipif(EIGEN is None or not os.path.isdir(REF_SRC),
                                reason="no real Eigen on disk (or no reference sources): Eigen's internals stay unpinned")


@pytest.fixture(scope="module")
def ref_eigen(oracle):
    subprocess.check_call(["make", "-C", os.path.join(ROOT, "oracle"), "-s", "ref_eigen", f"EIGEN={EIGEN}"])
    from oracle import reference as R
    saved = (R._SO, R._lib)
    R._SO, R._lib = os.path.join(ROOT, "oracle", "_ref", "libmadicp_ref_eigen.so"), None
    R.lib()
    yield R
    R._SO, R._lib = saved


def test_dot_order_discriminator(tmp_path):
    """(a0*b0 + a1*b1) + a2*b2 vs a0*b0 + (a1*b1 + a2*b2) differ in the last bit for this vector; the
    restatement defines the first (oracle dot3 / product arith.h)."""
    src = tmp_path / "dot.cpp"
    src.write_text('#include <Eigen/Core>\n#include <cstdio>\nint main(){volatile double e=1e-16;'
                   'Eigen::Vector3d a(1.0,e,e), b(1.0,1.0,1.0); std::printf("%a\\n", a.dot(b)); }\n')
    exe = tmp_path / "dot"
    subprocess.check_call(["g++", "-O3", "-DNDEBUG", "-std=c++17", f"-I{EIGEN}", str(src), "-o", str(exe)])
    got = float.fromhex(subprocess.check_output([str(exe)], text=True).strip())
    left, right = (1.0 + 1e-16) + 1e-16, 1.0 + (1e-16 + 1e-16)
    assert left != right
    assert got == left, "real Eigen reduces a 3-vector dot as a0b0 + (a1b1 + a2b2): flip dot3 in oracle and arith.h"


def test_tree_and_registration_bit_equal_to_real_eigen_build(oracle, ref_eigen):
    case = synth.registration_case(K=2, beams=16, azimuths=512)
    kfo, kfr = [], []
    for s in range(2):
        a, b = oracle.OracleTree(case["scans"][s]), ref_eigen.ReferenceTree(case["scans"][s])
        ea, eb = a.export(), b.export()
        for k in ea:
            assert np.array_equal(ea[k], eb[k], equal_nan=True), f"tree field {k} differs from the real-Eigen build"
        a.apply_transform(case["kf_poses"][s])
        b.apply_transform(case["kf_poses"][s])
        kfo.append(a)
        kfr.append(b)
    mo, mr = oracle.OracleTree(case["query"]), ref_eigen.ReferenceTree(case["query"])
    ro = oracle.icp_run(kfo, mo, case["T_guess"], iters=10, num_threads=2)
    rr = ref_eigen.icp_run(kfr, mr, case["T_guess"], iters=10, num_threads=2, record_idx=True)
    assert np.array_equal(np.asarray(ro["idx_hist"]), rr["idx_hist"])
    for k in ("X_hist", "H_hist", "b_hist", "X", "matched"):
        assert np.array_equal(ro[k], rr[k]), k
