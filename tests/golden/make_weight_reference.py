"""Writes keyframe_weight_reference.npz: the reference's keyframe weight on singular and near-singular H.

pipeline.cpp:223 weighs a frame by H_adder_.inverse().determinant(), and Pipeline keeps the frame with the smallest
weight as a keyframe (pipeline.cpp:234-241).  This library computes 1/det(H) instead.  The two differ where H is
singular, and there the difference decides which frame becomes a keyframe.  This script evaluates the reference's own
expression (oracle/ref_capi.cpp ref_inverse_determinant, the reference's Eigen calls compiled against
oracle/eigen_standin) on:
  kind 0: exactly singular H = P^T L D L^T P from dyadic factors (one zero in D).  Partial-pivot LU meets its only
          zero pivot at the last step, exactly, with a positive or a negative running product;
  kind 1: exactly singular H of the same family whose LU meets a zero pivot before the last step;
  kind 2: near-singular H, the kind-0 matrices with one diagonal entry moved by a few ulp: both libraries return
          rounding noise there, and only its finiteness is compared.
Run from the repository root after `make -C oracle ref`:  python tests/golden/make_weight_reference.py
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from oracle import reference as R  # noqa: E402


def lu_pivots(H):
    """Partial-pivot LU in float64 in solve6.h inv_det6's order: (pivots, running product)."""
    A = np.array(H, dtype=np.float64)
    det, piv = 1.0, []
    for k in range(6):
        p = k
        for i in range(k + 1, 6):
            if abs(A[i, k]) > abs(A[p, k]):
                p = i
        if p != k:
            A[[k, p]] = A[[p, k]]
            det = -det
        det = det * A[k, k]
        piv.append(A[k, k])
        for i in range(k + 1, 6):
            f = A[i, k] / A[k, k]
            for c in range(k, 6):
                A[i, c] = A[i, c] - f * A[k, c]
    return piv, det


def singular_cases(seed=11, want=(12, 12, 8)):
    rs = np.random.RandomState(seed)
    out = {0: [], 1: []}
    with np.errstate(all="ignore"):
        while len(out[0]) < want[0] + want[1] or len(out[1]) < want[2]:
            L = np.eye(6)
            for r in range(1, 6):
                for c in range(r):
                    if rs.rand() < 0.5:
                        L[r, c] = rs.choice([0.5, -0.5, 0.25, -0.25, 1.0, -1.0])
            D = 2.0 ** rs.randint(-2, 4, size=6)
            D[rs.randint(6)] = 0.0
            perm = rs.permutation(6)
            H = (L @ np.diag(D) @ L.T)[np.ix_(perm, perm)]
            piv, det = lu_pivots(H)
            zero = [k for k in range(6) if piv[k] == 0.0]
            if zero == [5] and all(np.isfinite(piv)):
                neg = np.signbit(det)
                n_neg = sum(np.signbit(lu_pivots(h)[1]) for h in out[0])
                if (neg and n_neg < want[0]) or (not neg and len(out[0]) - n_neg < want[1]):
                    out[0].append(H)
            elif zero and zero[0] < 5 and len(out[1]) < want[2]:
                out[1].append(H)
    return out


def main():
    cases = singular_cases()
    Hs, kinds = [], []
    for kind in (0, 1):
        for H in cases[kind]:
            Hs.append(H)
            kinds.append(kind)
    for j, H in enumerate(cases[0]):  # near-singular: one nonzero diagonal entry a few ulp away, no pivot zero
        Hn = H.copy()
        i = [k for k in range(6) if H[k, k] != 0][j % 5]
        for _ in range(1 + j % 3):
            Hn[i, i] = np.nextafter(Hn[i, i], np.inf)
        piv, _ = lu_pivots(Hn)
        if all(p != 0.0 for p in piv) and kinds.count(2) < 8:
            Hs.append(Hn)
            kinds.append(2)
    Hs = np.array(Hs)
    ref = np.array([R.inverse_determinant(H) for H in Hs])
    np.savez_compressed(os.path.join(HERE, "keyframe_weight_reference.npz"), H=Hs, kind=np.array(kinds, np.int32),
                        ref_weight=ref)
    print(f"{len(Hs)} cases; reference weight by kind:",
          {k: ref[np.array(kinds) == k].tolist() for k in (0, 1)})


if __name__ == "__main__":
    main()
