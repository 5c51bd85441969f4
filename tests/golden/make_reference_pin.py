"""Regenerates the stored outputs of the reference's own sources that the tests compare against:

  tests/golden/reference_pin.json     digests of every case of tests/test_reference_pin.py
  tests/golden/full16_reference.npz   the full-size registration of tests/test_gpu_parity.py (16 keyframes)

Needs oracle/_ref/libmadicp_ref.so: the reference's mad_tree.cpp, mad_icp.cpp, vel_estimator.cpp and pipeline.cpp
compiled against oracle/eigen_standin, built from a checkout of the reference with
`make -C oracle ref REF=<reference checkout>/mad_icp/src`.  Run it after changing a case or the synthetic inputs.
"""
import hashlib
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(HERE))
from mad_icp_b200 import synth  # noqa: E402
from oracle import reference as R  # noqa: E402
from util import digest  # noqa: E402
import test_reference_pin as T  # noqa: E402


def reference_backend():
    """The reference's own build behind the interface of the case functions (test_reference_pin.backend)."""
    return types.SimpleNamespace(Tree=R.ReferenceTree, icp_run=R.icp_run, Pipeline=R.ReferencePipeline,
                                 deskew=lambda pts, Ta, Tb: R.ReferencePipeline(deskew=True, num_threads=1).deskew(pts, Ta, Tb),
                                 idx_kw={"record_idx": True})


def full16():
    """registration_case(K=16) through the reference: its trees (std::async levels), its 10-round loop with its own
    correspondences.  The correspondences (10 x 16 x ~19k) are stored as one digest per round, plus a fixed seeded
    sample of 4096 of them per round (flat index into keyframe x leaf) so that a mismatch can be located."""
    c = synth.registration_case(K=16)
    trees = []
    for scan, P in zip(c["scans"], c["kf_poses"]):
        t = R.ReferenceTree(scan, max_parallel_level=2)
        t.apply_transform(P)
        trees.append(t)
    q = R.ReferenceTree(c["query"])
    r = R.icp_run(trees, q, c["T_guess"], iters=10, num_threads=min(16, R.max_threads()), record_idx=True)
    flat = r["idx_hist"].reshape(10, -1)
    pos = np.sort(np.random.RandomState(0).choice(flat.shape[1], 4096, replace=False)).astype(np.int32)
    np.savez_compressed(os.path.join(HERE, "full16_reference.npz"),
                        query_sha256=hashlib.sha256(c["query"].tobytes()).hexdigest(), X=r["X"], X_hist=r["X_hist"],
                        H_hist=r["H_hist"], b_hist=r["b_hist"], matched=np.packbits(r["matched"] != 0),
                        num_leaves=q.num_leaves, idx_shape=np.array(r["idx_hist"].shape),
                        idx_digest=np.array([digest(r["idx_hist"][it]) for it in range(10)]),
                        idx_sample_pos=pos, idx_sample=flat[:, pos])
    print("full16_reference: moving leaves", q.num_leaves)


def main():
    if not os.path.exists(R._SO):
        raise SystemExit(f"{R._SO} is missing: make -C oracle ref REF=<reference checkout>/mad_icp/src")
    R.lib()
    M = reference_backend()
    pinned = {}
    for name, (fn, kw) in T.CASES.items():
        pinned[name] = T.digests(fn(M, **kw))
        print(name, "ok")
    with open(T.GOLDEN, "w") as f:
        json.dump(pinned, f, indent=1, sort_keys=True)
    full16()


if __name__ == "__main__":
    main()
