"""Path memo modes of the persistent kernel, `-m gpu`: 0 walks every pair from the root in every round, 1 keeps the
leaves it proves unchanged, 2 (the default) also resumes the other walks from the deepest record of their last path it
proves unchanged (kernels.cuh, descend_t).  The proofs must be airtight: every mode returns the same bits."""
import numpy as np
import pytest

from mad_icp_b200 import FlatTree, MadIcpError, Registrar, synth
from util import bits_equal

pytestmark = pytest.mark.gpu

SMALL = dict(K=3, beams=32, azimuths=1024, seed=11)


def _registrar(c):
    reg = Registrar(device=0, max_keyframes=16)
    for k, (scan, P) in enumerate(zip(c["scans"], c["kf_poses"])):
        reg.put_keyframe(k, FlatTree(scan), T=P)
    reg.set_moving(FlatTree(c["query"]).leaf_means())
    return reg


def _run_modes(reg, X0, iters):
    out = []
    for mode in (0, 1, 2):
        reg.set_memo(mode)
        r = reg.register(X0, iters=iters)
        r["trace"] = reg.register_trace()
        r["walked"] = reg.register_walked()
        r["records"] = reg.register_walk_records()
        out.append(r)
    return out


def _assert_same(runs, what):
    a = runs[0]
    for mode, b in enumerate(runs[1:], start=1):
        for k in ("X", "H", "b", "trace"):
            assert bits_equal(a[k], b[k]), (what, mode, k)
        assert (a["matched"] == b["matched"]).all() and a["n_matched"] == b["n_matched"], (what, mode)


@pytest.mark.parametrize("kw", [SMALL, dict(K=16)], ids=["small", "baseline"])
def test_memo_modes_change_nothing(kw):
    """From the guess, from the guess 1.5 m off (large moves between rounds, many resumed walks), and from the optimum
    (nothing moves): poses, H, b, matched flags and the per-round trace bit-identical in modes 0, 1 and 2."""
    c = synth.registration_case(**kw)
    reg = _registrar(c)
    pairs = reg.num_keyframes * reg.L
    for shift in (0.0, 1.5):
        X0 = np.array(c["T_guess"], dtype=np.float64)
        X0[0, 3] += shift
        for iters in (1, 2, 10, 15):
            runs = _run_modes(reg, X0, iters)
            _assert_same(runs, (shift, iters))
            off, leaf, resume = runs
            assert (off["walked"] == pairs).all()
            # round 0 walks every pair from the root in every mode: the same records
            assert off["records"][0] == leaf["records"][0] == resume["records"][0]
            for r in runs:
                assert (r["records"] >= r["walked"]).all() and ((r["records"] == 0) == (r["walked"] == 0)).all()
    # restart from the converged pose: next to nothing moves, nearly every walk of rounds >= 1 is skipped
    runs = _run_modes(reg, runs[0]["X"], 5)
    _assert_same(runs, "optimum")
    reg.set_memo(True)


def test_set_memo_modes():
    """Booleans keep their meaning (True: the default mode 2, False: off); other modes are rejected."""
    c = synth.registration_case(K=1, beams=16, azimuths=512, seed=3)
    reg = _registrar(c)
    ref = reg.register(c["T_guess"], iters=4)
    for mode in (False, True, 0, 1, 2):
        reg.set_memo(mode)
        out = reg.register(c["T_guess"], iters=4)
        assert bits_equal(out["X"], ref["X"]), mode
    reg.set_memo(False)
    reg.register(c["T_guess"], iters=4)
    assert (reg.register_walked() == reg.num_keyframes * reg.L).all()
    for bad in (-1, 3):
        with pytest.raises(MadIcpError):
            reg.set_memo(bad)
