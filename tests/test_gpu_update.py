"""The Gauss-Newton update and the keyframe weight against exact arithmetic.

Every pose comes out of solve6.h: the pivoted LDL^T solve of H dx = -b (Eigen 3.4 LDLT<Matrix6d>, mad_icp.cpp:111),
Rodrigues' formula (lie_algebra.h:39-52) and X * dX.  Its keyframe weight det(H^-1) (pipeline.cpp:223) decides which
frame Pipeline keeps.  The exact reference below is written here from Eigen's published algorithm
(ldlt_inplace<Lower>::unblocked and LDLT::_solve_impl) in rational arithmetic and shares no code with solve6.h or the
oracle:
  * pivot: the largest |diagonal| among the remaining entries, the first maximum wins;
  * swap: row and column k with the pivot's, in the lower triangle;
  * update: A[k][k] -= sum_j A[k][j] D[j] A[k][j], and A21 likewise (left-looking);
  * a zero pivot at k = 0 stops the factorisation (the whole diagonal is zero); elsewhere it leaves A21 unscaled;
  * solve: P b, unit-lower solve, pseudo-inverse of D (|D_i| > DBL_MIN, else 0), unit-upper solve, P^T.
On a well-conditioned H every pivot order gives the same x to rounding, so the cases that can tell a wrong pivot order,
a wrong cut-off or a wrong index apart are the rank-deficient ones, the ties, and the exact ones: dyadic H whose every
intermediate is a float64, where the device must return the exact x bit for bit.

K3 (Registrar.solve_update) returns X * exp(dx), not dx.  With X = I and a right-hand side scaled by a power of two so
that theta^2 < 1e-8, the pose is [I + [w]x | t] and gives back all six components of dx exactly (a power-of-two scale
commutes with every rounding of the solve while nothing underflows).
"""
import math
import os
from fractions import Fraction as Fr
from itertools import permutations

import mpmath
import numpy as np
import pytest

from util import bits_equal

GOLD = os.path.join(os.path.dirname(__file__), "golden")
DBL_MIN = float(np.finfo(np.float64).tiny)
U = 2.0 ** -53  # unit roundoff
N = 6


def gamma(m):
    return m * U / (1.0 - m * U)


# ====================================================================== exact reference (rational arithmetic)
def _fr(v):
    return Fr(float(v))


def ldlt_factor(H, tie_last=False):
    """Eigen's LDLT::compute on the lower triangle of H, exactly.  tie_last: the last maximal diagonal wins (a
    deliberately wrong tie-break, used to find the cases that tell the two apart).  Returns A (L below the diagonal,
    D on it, pivot frame), the transpositions, whether the factorisation stopped at k = 0, and every intermediate value
    the left-looking order produces (products and partial sums)."""
    A = [[_fr(H[r][c]) if r >= c else None for c in range(N)] for r in range(N)]
    tr, vals = list(range(N)), []
    for k in range(N):
        big = k
        for i in range(k + 1, N):
            a, m = abs(A[i][i]), abs(A[big][big])
            if a > m or (tie_last and a == m):
                big = i
        tr[k] = big
        if big != k:
            for j in range(k):
                A[k][j], A[big][j] = A[big][j], A[k][j]
            for i in range(big + 1, N):
                A[i][k], A[i][big] = A[i][big], A[i][k]
            A[k][k], A[big][big] = A[big][big], A[k][k]
            for i in range(k + 1, big):
                A[i][k], A[big][i] = A[big][i], A[i][k]
        if k > 0:
            w = [A[j][j] * A[k][j] for j in range(k)]
            vals += w
            for i in range(k, N):
                s = Fr(0)
                for j in range(k):
                    p = A[i][j] * w[j]
                    s += p
                    vals += [p, s]
                A[i][k] -= s
                vals.append(A[i][k])
        d = A[k][k]
        if k == 0 and d == 0:
            return dict(A=A, tr=list(range(N)), stopped=True, vals=vals)
        if d != 0:
            if abs(d) > Fr(DBL_MIN):
                vals.append(1 / d)
            for i in range(k + 1, N):
                A[i][k] /= d
                vals.append(A[i][k])
    return dict(A=A, tr=tr, stopped=False, vals=vals)


def ldlt_solve(f, b):
    """Eigen's LDLT::_solve_impl for the right-hand side -b, exactly: (x, intermediate values)."""
    A, tr, vals = f["A"], f["tr"], []
    y = [-_fr(v) for v in b]
    for k in range(N):
        y[k], y[tr[k]] = y[tr[k]], y[k]
    for i in range(N):
        for j in range(i):
            p = A[i][j] * y[j]
            y[i] -= p
            vals += [p, y[i]]
    for i in range(N):
        y[i] = y[i] / A[i][i] if abs(A[i][i]) > Fr(DBL_MIN) else Fr(0)
        vals.append(y[i])
    for i in reversed(range(N)):
        for j in range(i + 1, N):
            p = A[j][i] * y[j]
            y[i] -= p
            vals += [p, y[i]]
    for k in reversed(range(N)):
        y[k], y[tr[k]] = y[tr[k]], y[k]
    return y, vals


def pivot_order(f):
    order = list(range(N))
    for k in range(N):
        order[k], order[f["tr"][k]] = order[f["tr"][k]], order[k]
    return order


def factors(f):
    """(L unit lower, D) in the pivot frame."""
    A = f["A"]
    L = [[Fr(1) if r == c else (A[r][c] if r > c and not f["stopped"] else Fr(0)) for c in range(N)] for r in range(N)]
    D = [A[i][i] if not f["stopped"] else Fr(0) for i in range(N)]
    return L, D


def is_double(q):
    try:
        v = float(q)
    except OverflowError:
        return False
    return math.isfinite(v) and Fr(v) == q


def is_pow2(q):
    q = abs(q)
    return q.numerator & (q.numerator - 1) == 0 and q.denominator & (q.denominator - 1) == 0


def det_bareiss(H):
    """Exact determinant (fraction-free Bareiss elimination over the rationals, row exchanges on zero pivots)."""
    M = [[_fr(H[r][c]) for c in range(N)] for r in range(N)]
    sign, prev = 1, Fr(1)
    for k in range(N - 1):
        if M[k][k] == 0:
            sw = next((i for i in range(k + 1, N) if M[i][k] != 0), None)
            if sw is None:
                return Fr(0)
            M[k], M[sw] = M[sw], M[k]
            sign = -sign
        for i in range(k + 1, N):
            for j in range(k + 1, N):
                M[i][j] = (M[i][j] * M[k][k] - M[i][k] * M[k][j]) / prev
        prev = M[k][k]
    return sign * M[N - 1][N - 1]


def solve_exact(M, rhs):
    """Exact Gauss-Jordan: M^-1 rhs for a nonsingular rational M (rhs: list of columns)."""
    A = [row[:] + [c[i] for c in rhs] for i, row in enumerate(M)]
    n, m = len(M), len(rhs)
    for k in range(n):
        p = next(i for i in range(k, n) if A[i][k] != 0)
        A[k], A[p] = A[p], A[k]
        piv = A[k][k]
        A[k] = [v / piv for v in A[k]]
        for i in range(n):
            if i != k and A[i][k] != 0:
                f = A[i][k]
                A[i] = [a - f * c for a, c in zip(A[i], A[k])]
    return [[A[i][n + j] for i in range(n)] for j in range(m)]


def sym_lower(H):
    """The symmetric matrix the solve sees: the lower triangle of H mirrored."""
    H = np.asarray(H, dtype=np.float64)
    return np.tril(H) + np.tril(H, -1).T


def rodrigues_exact(w, prec=256):
    """exp([w]x) at `prec` bits (mpmath), for the float64 vector w taken exactly."""
    with mpmath.workprec(prec):
        wx, wy, wz = (mpmath.mpf(float(v)) for v in w)
        th = mpmath.sqrt(wx * wx + wy * wy + wz * wz)
        W = mpmath.matrix([[0, -wz, wy], [wz, 0, -wx], [-wy, wx, 0]])
        R = mpmath.eye(3) + (mpmath.sin(th) / th) * W + ((1 - mpmath.cos(th)) / (th * th)) * (W * W)
        return R, th


# ====================================================================== the kernel's observable: dx through K3
def th2_of(w):
    """theta^2 as expmap_so3 rounds it: dot3 order (x*x + y*y) + z*z, no FMA (Python floats are IEEE doubles)."""
    x, y, z = (float(v) for v in w)
    return (x * x + y * y) + z * z


def pose_from_dx(dx, small_branch=True):
    """The pose K3 returns for X = I when theta^2 < 1e-8: iso_mul(I, [I + [w]x | t]) in arith.h's order."""
    t, (wx, wy, wz) = [float(v) for v in dx[:3]], [float(v) for v in dx[3:]]
    assert th2_of((wx, wy, wz)) < 1e-8 or not small_branch
    W = [0.0, -wz, wy, wz, 0.0, -wx, -wy, wx, 0.0]
    R = [(1.0 if i % 4 == 0 else 0.0) + W[i] for i in range(9)]
    B = [R[0], R[1], R[2], t[0], R[3], R[4], R[5], t[1], R[6], R[7], R[8], t[2]]
    I = [1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 0.0, 1.0, 0.0]
    out = np.empty((3, 4))
    for r in range(3):
        a = I[r * 4:r * 4 + 3]
        for c in range(3):
            out[r, c] = (a[0] * B[c] + a[1] * B[4 + c]) + a[2] * B[8 + c]
        out[r, 3] = ((a[0] * B[3] + a[1] * B[7]) + a[2] * B[11]) + I[r * 4 + 3]
    return out


def rhs_scale(x_max):
    """A power of two 2^-s that brings max |dx| to <= 2^-17, so theta^2 < 1e-8 with room (s >= 0)."""
    if not x_max > 0:
        return 1.0
    return 2.0 ** -max(0, math.frexp(x_max)[1] + 17)


def k3_dx(reg, H, b, x_max):
    """dx as K3 computes it for (H, b): solve (H, sc*b) at X = I and read [t | w] off the pose, then undo sc."""
    sc = rhs_scale(x_max)
    Xn = reg.solve_update(np.asarray(H, np.float64), np.asarray(b, np.float64) * sc, np.eye(4)[:3])
    w = (Xn[2, 1], Xn[0, 2], Xn[1, 0])
    assert th2_of(w) < 1e-8 and bits_equal(Xn, pose_from_dx(list(Xn[:, 3]) + list(w))), Xn
    return np.array(list(Xn[:, 3]) + list(w)) / sc, Xn, sc


# ====================================================================== case families
def _rand_unit_lower(rs, entries=(0.5, -0.5, 0.25, -0.25, 1.0, -1.0), density=0.5):
    L = np.eye(N)
    for r in range(1, N):
        for c in range(r):
            if rs.rand() < density:
                L[r, c] = rs.choice(entries)
    return L


def _exact_ok(H, b):
    f = ldlt_factor(H)
    x, sv = ldlt_solve(f, b)
    _, D = factors(f)
    ok = all(is_double(v) for v in f["vals"] + sv + x) and all(d == 0 or is_pow2(d) for d in D)
    return ok, f, x


def _dyadic_rhs(rs):
    return rs.choice([1.0, -1.0, 0.5, -0.5, 2.0, -2.0, 0.25, 0.0, 3.0], size=N)


def full_rank_bases(n_bases=6, seed=1):
    """Dyadic B = L D L^T with a distinct diagonal whose own factorisation is exact with power-of-two pivots."""
    rs, out = np.random.RandomState(seed), []
    while len(out) < n_bases:
        L = _rand_unit_lower(rs)
        D = 2.0 ** rs.randint(-2, 5, size=N)
        B = L @ np.diag(D) @ L.T
        if len(set(np.abs(np.diag(B)))) < N:
            continue
        ok, f, _ = _exact_ok(B, np.ones(N))
        if ok and all(d != 0 for d in factors(f)[1]):
            out.append(B)
    return out


def exact_cases():
    """(name, H, b) with the exact x a float64 vector and every intermediate a float64: all 720 pivot orders of a
    distinct diagonal at full rank, every rank 0..5 with a zero pivot at every position 1..5, and ties of 2..6
    maximal diagonals whose tie-break changes x."""
    rs = np.random.RandomState(2)
    cases = []
    bases = full_rank_bases()
    for i, perm in enumerate(permutations(range(N))):
        B = bases[i % len(bases)]
        H = B[np.ix_(perm, perm)]
        b = _dyadic_rhs(rs)
        ok, f, _ = _exact_ok(H, b)
        if not ok:  # a right-hand side that rounds: keep the order, use a plainer b
            b = np.ones(N)
            ok, f, _ = _exact_ok(H, b)
        assert ok and pivot_order(f) == sorted(range(N), key=lambda j: -abs(H[j, j])), perm
        cases.append((f"order{perm}", H, b))
    # ranks: H = G G^T with G of {0, +-1} entries and r columns, and L D L^T with zeros in D
    seen = set()
    want = {(r, k) for r in range(1, N) for k in range(1, N)}
    tries = 0
    while (want - seen) and tries < 200000:
        tries += 1
        r = rs.randint(1, N)
        if rs.rand() < 0.5:
            G = rs.choice([0.0, 0.0, 1.0, -1.0], size=(N, r))
            H = G @ G.T
        else:
            L = _rand_unit_lower(rs)
            D = 2.0 ** rs.randint(-2, 4, size=N)
            D[rs.choice(N, N - r, replace=False)] = 0.0
            H = (L @ np.diag(D) @ L.T)[np.ix_(*(2 * [rs.permutation(N)]))]
        b = _dyadic_rhs(rs)
        ok, f, _ = _exact_ok(H, b)
        if not ok or f["stopped"]:
            continue
        D = factors(f)[1]
        rank = sum(d != 0 for d in D)
        new = {(rank, k) for k in range(1, N) if D[k] == 0} - seen
        if new:
            seen |= new
            cases.append((f"rank{rank}_zero{sorted(k for k in range(N) if D[k] == 0)}", H, b))
    assert not (want - seen), f"no exact case for (rank, zero pivot position) {sorted(want - seen)}"
    cases.append(("rank0", np.zeros((N, N)), _dyadic_rhs(rs)))
    # ties of the maximal |diagonal| that the first-maximum rule resolves differently from the last-maximum one
    ties = {m: 0 for m in range(2, N + 1)}
    tries = 0
    while min(ties.values()) < 3 and tries < 400000:
        tries += 1
        G = rs.choice([0.0, 0.0, 1.0, -1.0], size=(N, rs.randint(1, N)))
        H = G @ G.T
        dg = np.abs(np.diag(H))
        m = int((dg == dg.max()).sum())
        if dg.max() == 0 or m < 2 or ties[m] >= 3:
            continue
        b = _dyadic_rhs(rs)
        ok, f, x = _exact_ok(H, b)
        if not ok:
            continue
        x_last, _ = ldlt_solve(ldlt_factor(H, tie_last=True), b)
        if x_last != x:
            ties[m] += 1
            cases.append((f"tie{m}_{ties[m]}", H, b))
    assert min(ties.values()) >= 3, ties
    return cases


def tolerance_cases():
    """(name, H, b, which component, kept?) around the pseudo-inverse's cut-off |D_i| > DBL_MIN."""
    out = []
    nxt = float(np.nextafter(DBL_MIN, np.inf))
    for d, kept in ((DBL_MIN, False), (-DBL_MIN, False), (nxt, True), (-nxt, True), (DBL_MIN / 2, False),
                    (2.0 ** -1074, False), (-(2.0 ** -1060), False), (0.0, False), (-0.0, False)):
        for comp in (0, 2):
            H = np.eye(N)
            H[comp, comp] = d
            b = -np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0])
            out.append((f"d={d!r}@{comp}", H, b, comp, kept))
    # a subnormal pivot that is not the last one, over a column of zeros: Eigen divides 0 by it
    for sub in (2.0 ** -1074, 2.0 ** -1040):
        H = np.diag([1.0, 1.0, 1.0, 1.0, sub, 0.0])
        H[:, [0, 4]] = H[:, [4, 0]]
        H[[0, 4], :] = H[[4, 0], :]
        out.append((f"subnormal {sub!r} before a zero pivot", H, -np.array([1.0, 1.0, 1.0, 0.0, 0.0, 0.0]), 0, False))
    return out


def special_zero_cases():
    return [("all zero", np.zeros((N, N)), np.ones(N)), ("all -0.0", np.full((N, N), -0.0), np.ones(N)),
            ("-0.0 diagonal", np.diag([1.0, -0.0, 2.0, -0.0, 0.5, 4.0]), np.ones(N))]


def jacobian_cases():
    """(name, H, b, kappa) from this path's own Jacobian rows J = n^T [I | -skew(p)], folded as the kernel folds them:
    H[r][c] += (s J_r) J_c with a Huber-like weight s, b += (s J) e.  Normals clustered around one direction set the
    conditioning: kappa from ~1 to ~1e12."""
    rs = np.random.RandomState(7)
    out = []
    for spread in (1.0, 0.3, 1e-1, 3e-2, 1e-2, 3e-3, 1e-3, 3e-4, 1e-4, 3e-5, 1e-5, 3e-6, 1e-6):
        n = 200
        P = rs.uniform(-20, 20, size=(n, 3))
        nrm = np.array([0.0, 0.0, 1.0]) + spread * rs.randn(n, 3)
        if spread >= 1.0:
            nrm = rs.randn(n, 3)
        nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
        e = rs.randn(n) * 0.05
        H, b = np.zeros((N, N)), np.zeros(N)
        for p, q, ei in zip(P, nrm, e):
            sk = np.array([[0, -p[2], p[1]], [p[2], 0, -p[0]], [-p[1], p[0], 0]])
            J = np.concatenate([q, -(q @ sk)])
            s = 1.0 if abs(ei) < 0.1 else 0.1 / abs(ei)
            sJ = s * J
            for r in range(N):
                for c in range(N):
                    H[r, c] += sJ[r] * J[c]
                b[r] += sJ[r] * ei
        Hs = sym_lower(H)
        out.append((f"jacobian spread={spread}", H, b, float(np.linalg.cond(Hs, np.inf))))
    return out


def golden_cases():
    out = []
    for name in ("lidar_small_registration", "four_walls_registration"):
        g = np.load(os.path.join(GOLD, name + ".npz"))
        for it in range(g["H_hist"].shape[0]):
            out.append((f"{name}[{it}]", g["H_hist"][it], g["b_hist"][it], None))
    return out


def rounded_bar(H, b, xh):
    """Backward-error bar of the rounded solve: |H x^ + b| <= g (|P^T L| |D| |L^T P| |x^| + |b|), componentwise, with
    exact L, D of the lower triangle of H.  g = 2 gamma_{3n+4}, n = 6:
      factorisation  gamma_{n+2}: inner products of <= n-1 terms, the product D_j L_kj, and the pivot's reciprocal
                     (solve6.h multiplies by 1/d where Eigen divides: two roundings instead of one);
      forward and back substitution  gamma_{n-1} each;  scaling by the pseudo-inverse  gamma_2 (reciprocal, product);
    summed to first order that is gamma_{3n+2}; 2 more for the sums of the bound itself, and the factor 2 covers the
    difference between the exact factors used here and the computed ones the theorem is stated with (for a PSD H
    both are bounded by sqrt(H_ii H_jj), by Cauchy-Schwarz on sum_j L_ij^2 D_j = H_ii).  The bar does not depend on
    the condition number.  Returns (max violation ratio, the forward-error bar's gamma' = n g)."""
    Hs = sym_lower(H)
    f = ldlt_factor(Hs)
    L, D = factors(f)
    order = pivot_order(f)
    g = 2 * gamma(3 * N + 4)
    LDL = [[sum(abs(L[i][k]) * abs(D[k]) * abs(L[j][k]) for k in range(N)) for j in range(N)] for i in range(N)]
    inv = [0] * N
    for i, o in enumerate(order):
        inv[o] = i
    xq = [_fr(v) for v in xh]
    worst = 0.0
    for r in range(N):
        res = sum(_fr(Hs[r, c]) * xq[c] for c in range(N)) + _fr(b[r])
        bound = sum(LDL[inv[r]][inv[c]] * abs(xq[c]) for c in range(N)) + abs(_fr(b[r]))
        if res != 0:
            worst = max(worst, float(abs(res) / (g * bound)) if bound > 0 else math.inf)
    return worst, N * g


def forward_error(H, b, xh):
    """(||x^ - x||_inf / ||x||_inf, kappa_inf(H)) with x and H^-1 exact."""
    Hs = sym_lower(H)
    M = [[_fr(Hs[r, c]) for c in range(N)] for r in range(N)]
    cols = solve_exact(M, [[-_fr(v) for v in b]] + [[Fr(int(i == j)) for i in range(N)] for j in range(N)])
    x, Hinv = cols[0], cols[1:]
    nH = max(sum(abs(M[r][c]) for c in range(N)) for r in range(N))
    nHi = max(sum(abs(Hinv[c][r]) for c in range(N)) for r in range(N))
    err = max(abs(_fr(xh[i]) - x[i]) for i in range(N)) / max(abs(v) for v in x)
    return float(err), float(nH * nHi)


def nan_inf_cases():
    nan, inf = float("nan"), float("inf")
    out = []
    base = np.diag([4.0, 2.0, 1.0, 0.5, 8.0, 0.25])
    base[3, 1] = base[1, 3] = 0.5
    base[5, 0] = base[0, 5] = -1.0
    for (r, c) in ((0, 0), (2, 2), (3, 1), (5, 0), (5, 5), (4, 2)):
        for v in (nan, inf, -inf):
            H = base.copy()
            H[r, c] = v
            if r != c:
                H[c, r] = v
            out.append((f"H[{r},{c}]={v}", H, np.ones(N)))
    rank_def = np.diag([1.0, 1.0, 1.0, 1.0, 1.0, 0.0])
    for (i, v) in ((5, inf), (5, nan), (0, inf), (0, nan)):
        b = np.ones(N)
        b[i] = v
        out.append((f"b[{i}]={v} on diag(1,1,1,1,1,0)", rank_def, b))
    H = np.eye(N)
    H[0, 0] = nan
    out.append(("H[0,0]=nan, rest identity", H, np.ones(N)))
    out.append(("all nan", np.full((N, N), nan), np.ones(N)))
    H = np.zeros((N, N))
    H[3, 1] = H[1, 3] = inf
    out.append(("zero diagonal, inf below it", H, np.ones(N)))
    return out


@pytest.fixture(scope="module")
def exact():
    return exact_cases()


@pytest.fixture(scope="module")
def reg(built):
    from mad_icp_b200 import Registrar
    return Registrar(device=0, max_keyframes=2)


def _kind(a):
    a = np.asarray(a, np.float64)
    return np.where(np.isnan(a), 0, np.where(np.isposinf(a), 1, np.where(np.isneginf(a), 2, 3)))


# ====================================================================== CPU: the exact reference against the oracle
def test_exact_reference_is_a_factorisation(exact):
    """The reference itself: P^T L D L^T P reproduces H, and x solves H x = -b where H is nonsingular."""
    for name, H, b in exact[::23]:
        f = ldlt_factor(H)
        L, D = factors(f)
        order = pivot_order(f)
        for i in range(N):
            for j in range(i + 1):
                assert sum(L[i][k] * D[k] * L[j][k] for k in range(N)) == _fr(H[order[i], order[j]]), name
        if all(d != 0 for d in D):
            x, _ = ldlt_solve(f, b)
            for r in range(N):
                assert sum(_fr(H[r, c]) * x[c] for c in range(N)) == -_fr(b[r]), name


def test_oracle_exact_cases(exact, oracle):
    for name, H, b in exact:
        x, _ = ldlt_solve(ldlt_factor(H), b)
        dx, _ = oracle.solve_update(H, b, np.eye(4))
        assert bits_equal(dx + 0.0, np.array([float(v) for v in x]) + 0.0), (name, dx, [float(v) for v in x])


def test_oracle_tolerance_edge_and_zeros(oracle):
    for name, H, b, comp, kept in tolerance_cases():
        dx, _ = oracle.solve_update(H, b, np.eye(4))
        want = 1.0 / H[comp, comp] if kept else 0.0  # y = -b = 1 at the pivot; Eigen divides
        assert dx[comp] == want and np.isfinite(dx).all(), (name, dx)
    for name, H, b in special_zero_cases():
        x, _ = ldlt_solve(ldlt_factor(H), b)
        dx, _ = oracle.solve_update(H, b, np.eye(4))
        assert bits_equal(dx + 0.0, np.array([float(v) for v in x]) + 0.0), (name, dx)


def test_oracle_rounded_cases(oracle):
    for name, H, b, _ in jacobian_cases() + golden_cases():
        dx, _ = oracle.solve_update(H, b, np.eye(4))
        worst, g1 = rounded_bar(H, b, dx)
        assert worst <= 1.0, (name, worst)
        err, kappa = forward_error(H, b, dx)
        assert err <= kappa * g1 / max(1e-3, 1 - kappa * g1), (name, err, kappa)


def test_oracle_reads_the_lower_triangle_only(exact, oracle):
    for name, H, b in exact[::37] + [c[:3] for c in jacobian_cases()]:
        want, _ = oracle.solve_update(sym_lower(H), b, np.eye(4))
        for fill in (np.nan, 1e300):
            Hu = np.array(H, np.float64)
            Hu[np.triu_indices(N, 1)] = fill
            got, _ = oracle.solve_update(Hu, b, np.eye(4))
            assert bits_equal(got, want), (name, fill)


def test_identity_solve_returns_minus_b(oracle):
    """H = I: every pivot is 1 and every elimination term is 0 * something, so x = -b exactly.  This is what the
    exponential-map tests below rely on to drive expmap_so3 with a chosen dx."""
    rs = np.random.RandomState(3)
    for _ in range(50):
        b = rs.randn(N) * 10.0 ** rs.uniform(-8, 2)
        dx, _ = oracle.solve_update(np.eye(N), b, np.eye(4))
        assert bits_equal(dx, -b)


def test_oracle_weight_matches_exact_determinant(exact, oracle):
    for name, H, _ in exact[::7]:
        d = det_bareiss(H)
        w = oracle.inverse_determinant(H)
        if d != 0 and all(p != 0 for p in _lu_exact(H)[0]):
            assert w == float(1 / d) or abs(Fr(w) * d - 1) <= _weight_bar(H), (name, w, float(1 / d))


# ====================================================================== weight: exact bound
def _lu_exact(H):
    """Partial-pivot LU of H over the rationals with the same first-maximum row choice: (U diagonal, |L||U|)."""
    A = [[_fr(H[r][c]) for c in range(N)] for r in range(N)]
    Lm = [[Fr(0)] * N for _ in range(N)]
    perm = list(range(N))
    for k in range(N):
        p = k
        for i in range(k + 1, N):
            if abs(A[i][k]) > abs(A[p][k]):
                p = i
        A[k], A[p] = A[p], A[k]
        Lm[k], Lm[p] = Lm[p], Lm[k]
        perm[k], perm[p] = perm[p], perm[k]
        Lm[k][k] = Fr(1)
        if A[k][k] == 0:
            return [A[i][i] for i in range(N)], None
        for i in range(k + 1, N):
            f = A[i][k] / A[k][k]
            Lm[i][k] = f
            for c in range(k, N):
                A[i][c] -= f * A[k][c]
    LU = [[sum(abs(Lm[i][k]) * abs(A[k][j]) for k in range(N)) for j in range(N)] for i in range(N)]
    return [A[i][i] for i in range(N)], (LU, perm)


def _weight_bar(H):
    """|w/w_exact - 1| for w = 1/det(H) by partial-pivot LU.  The computed U is the exact one of H + E with
    |E| <= gamma_n P^T|L||U| (n = 6, elimination and division), and the product of the six pivots and the final
    reciprocal add gamma_{n+1}.  det(H + E)/det(H) = det(I + H^-1 E) lies within (1 +- eps)^n of 1 with
    eps = || |H^-1| gamma_n P^T |L||U| ||_inf.  So |w/w_exact - 1| <= rho/(1 - rho) with
    rho = (1 + eps)^n (1 + gamma_{n+1}) - 1; 2x for exact versus computed factors.  Returns None where rho >= 1/2:
    there det is below the LU's error and the weight is noise."""
    _, fac = _lu_exact(H)
    if fac is None:
        return None
    LU, perm = fac
    M = [[_fr(H[r][c]) for c in range(N)] for r in range(N)]
    Hinv = solve_exact(M, [[Fr(int(i == j)) for i in range(N)] for j in range(N)])  # columns
    E = [[0] * N for _ in range(N)]
    for i in range(N):
        E[perm[i]] = [v * Fr(gamma(N)) for v in LU[i]]
    eps = max(sum(abs(Hinv[k][r]) * E[k][c] for k in range(N) for c in range(N)) for r in range(N))
    rho = (1 + float(eps)) ** N * (1 + gamma(N + 1)) - 1
    if rho >= 0.5:
        return None
    return Fr(2 * rho / (1 - rho))


# ====================================================================== GPU: K3
@pytest.mark.gpu
def test_k3_exact_cases_bit_for_bit(exact, reg):
    for name, H, b in exact:
        x, _ = ldlt_solve(ldlt_factor(H), b)
        xf = np.array([float(v) for v in x])
        sc = rhs_scale(np.abs(xf).max())
        Xn = reg.solve_update(H, b * sc, np.eye(4)[:3])
        assert bits_equal(Xn, pose_from_dx(xf * sc)), (name, Xn, xf * sc)


@pytest.mark.gpu
def test_k3_tolerance_edge_and_zeros(reg):
    for name, H, b, comp, kept in tolerance_cases():
        Xn = reg.solve_update(H, b, np.eye(4)[:3])
        want = (1.0 / H[comp, comp]) * 1.0 if kept else 0.0  # y = 1 times the pivot's reciprocal
        assert np.isfinite(Xn).all() and Xn[comp, 3] == want, (name, Xn)
        assert bits_equal(Xn[:, :3], np.eye(3)), name
    for name, H, b in special_zero_cases():
        x, _ = ldlt_solve(ldlt_factor(H), b)
        xf = np.array([float(v) for v in x])
        sc = rhs_scale(np.abs(xf).max())
        assert bits_equal(reg.solve_update(H, b * sc, np.eye(4)[:3]), pose_from_dx(xf * sc)), name


@pytest.mark.gpu
def test_k3_rounded_cases(reg, oracle):
    for name, H, b, _ in jacobian_cases() + golden_cases():
        xo, _ = oracle.solve_update(H, b, np.eye(4))
        dx, _, _ = k3_dx(reg, H, b, np.abs(xo).max())
        worst, g1 = rounded_bar(H, b, dx)
        assert worst <= 1.0, (name, worst)
        err, kappa = forward_error(H, b, dx)
        assert err <= kappa * g1 / max(1e-3, 1 - kappa * g1), (name, err, kappa)


@pytest.mark.gpu
def test_k3_reads_the_lower_triangle_only(exact, reg):
    for name, H, b in exact[::37] + [c[:3] for c in jacobian_cases()]:
        want = reg.solve_update(sym_lower(H), b * 2.0 ** -40, np.eye(4)[:3])
        for fill in (np.nan, 1e300, "transpose-rounded"):
            Hu = np.array(H, np.float64)
            if fill == "transpose-rounded":  # an upper triangle that differs from the lower one by rounding
                Hu[np.triu_indices(N, 1)] *= 1.0 + 2.0 ** -40
            else:
                Hu[np.triu_indices(N, 1)] = fill
            assert bits_equal(reg.solve_update(Hu, b * 2.0 ** -40, np.eye(4)[:3]), want), (name, fill)


@pytest.mark.gpu
def test_k3_nan_and_inf_agree_with_the_oracle(reg, oracle):
    """The same class (NaN, +inf, -inf, finite) in every entry of the pose as the oracle, which divides where
    solve6.h multiplies by a reciprocal; finite entries agree to rounding."""
    for name, H, b in nan_inf_cases():
        with np.errstate(all="ignore"):
            _, Xo = oracle.solve_update(H, b, np.eye(4))
        Xd = reg.solve_update(H, b, np.eye(4)[:3])
        assert (_kind(Xd) == _kind(Xo)).all(), (name, Xd, Xo)
        fin = np.isfinite(Xo)
        assert np.all(np.abs(Xd[fin] - Xo[fin]) <= 1e-12 * np.maximum(1.0, np.abs(Xo[fin]))), (name, Xd, Xo)


# ====================================================================== GPU: exponential map and pose product
def _branch_vectors():
    """w with theta^2, as expmap_so3 rounds it, at 1e-8 exactly and 1, 2 and 1000 ulp either side."""
    T = 1e-8
    targets = {0: T}
    for k in (1, 2, 1000):
        up, dn = T, T
        for _ in range(k):
            up, dn = float(np.nextafter(up, 1.0)), float(np.nextafter(dn, 0.0))
        targets[k], targets[-k] = up, dn
    out = {}
    a0 = math.sqrt(T)
    for k, t in targets.items():
        found = None
        for da in range(-3000, 3000):
            a = a0 * (1.0 + da * 2.0 ** -52)
            aa = a * a
            if aa > t:
                continue
            for c in (0.0, 1e-13, 2e-13, 3e-13, 5e-13, 7e-13, 1e-12, 1.3e-12, 1.7e-12, 2e-12, 3e-12):
                if (aa + c * c) == t:
                    found = (a, c)
                    break
            if found:
                break
        assert found, k
        out[k] = found
    return out


@pytest.mark.gpu
def test_expmap_branch_at_theta2_1e8(reg, oracle):
    vecs = _branch_vectors()
    for k, (a, c) in vecs.items():
        for w in ((a, c, 0.0), (-c, 0.0, -a), (0.0, -a, c)):
            th2 = th2_of(w)
            assert th2 == 1e-8 if k == 0 else (th2 > 1e-8) == (k > 0), (k, w)
            dx = np.array([0.0, 0.0, 0.0, *w])
            Xn = reg.solve_update(np.eye(N), -dx, np.eye(4)[:3])
            if th2 < 1e-8:
                assert bits_equal(Xn, pose_from_dx(dx)), (k, w)
            else:
                R, _ = rodrigues_exact(w)
                assert not bits_equal(Xn, pose_from_dx(dx, small_branch=False)), (k, w)
                err = max(abs(mpmath.mpf(float(Xn[i, j])) - R[i, j]) for i in range(3) for j in range(3))
                assert err <= 8 * U, (k, w, float(err))
            _, Xo = oracle.solve_update(np.eye(N), -dx, np.eye(4))
            assert (th2 < 1e-8) == bits_equal(Xo, pose_from_dx(dx, small_branch=False)), (k, w)


def rotation_bar(theta):
    """Elementwise |R^ - R| for expmap_so3 at angle theta (u = 2^-53; CUDA's sin is within 2 ulp, <= 4u relative):
      theta^2 = (x^2 + y^2) + z^2: 3u relative;  theta = sqrt: 2.5u;  1/theta: 3.5u;  K = W/theta: eK = 4.5u;
      s = sin(theta):  e_s <= 2.5u theta |cos theta| + 4u |sin theta|;
      h = sin(theta/2): e_h <= 2.5u (theta/2) cos(theta/2) + 4u h;  omc = 2 h h: e_omc <= 4 h e_h + 2u omc;
      R = (I + s K) + (omc K) K: |K| <= 1 elementwise and sum_j |K_rj K_jc| <= 1, so
      |R^ - R| <= e_s + |s| (eK + u) + e_omc + omc (2 eK + 3u) + 2u (1 + |s| + omc),
    which is at most ~58u (about 29 ulp of 1) at theta = pi and a few ulp at small angles."""
    s, c = abs(math.sin(theta)), abs(math.cos(theta))
    h, ch = abs(math.sin(theta / 2)), abs(math.cos(theta / 2))
    omc = 2 * h * h
    eK = 4.5 * U
    e_s = 2.5 * U * theta * c + 4 * U * s
    e_h = 2.5 * U * (theta / 2) * ch + 4 * U * h
    e_omc = 4 * h * e_h + 2 * U * omc
    return (e_s + s * (eK + U) + e_omc + omc * (2 * eK + 3 * U) + 2 * U * (1 + s + omc)) * (1 + 1e-6)


def _angle_cases():
    rs = np.random.RandomState(9)
    thetas = list(np.geomspace(1.0001e-4, math.pi, 40)) + [3.0, 2 * math.pi - 1e-3, 2 * math.pi - 1e-9, math.pi]
    out = []
    for th in thetas:
        axis = rs.randn(3)
        axis /= np.linalg.norm(axis)
        out.append(axis * th)
    out += [np.array([math.pi, 0, 0]), np.array([0, 0, -3.0]), np.array([0, 2 * math.pi - 1e-6, 0])]
    return out


@pytest.mark.gpu
def test_expmap_rotation_against_exact_rodrigues(reg, oracle):
    for w in _angle_cases():
        dx = np.array([0.0, 0.0, 0.0, *w])
        Rd = reg.solve_update(np.eye(N), -dx, np.eye(4)[:3])[:, :3]  # X = I: the pose's rotation is exp(w) exactly
        Ro = oracle.solve_update(np.eye(N), -dx, np.eye(4))[1][:, :3]
        R, th = rodrigues_exact(w)
        bar = rotation_bar(float(th))
        for Rx in (Rd, Ro):
            err = max(abs(mpmath.mpf(float(Rx[i, j])) - R[i, j]) for i in range(3) for j in range(3))
            assert err <= bar, (w, float(err), bar)
            RtR = [[sum(Fr(float(Rx[k, i])) * Fr(float(Rx[k, j])) for k in range(3)) - int(i == j) for j in range(3)]
                   for i in range(3)]
            assert max(abs(float(v)) for row in RtR for v in row) <= 6 * bar + 4 * U, w
        assert np.abs(Rd - Ro).max() <= 2 * bar, w


@pytest.mark.gpu
def test_pose_product_at_world_scale(reg):
    """X * dX for X with |t| up to 1e4 m, against the exact product of X (exact doubles) with exp(w) and t:
    rotation entries within sum_k |RX_rk| (bar + gamma_3 |dR_kc|), translation within
    gamma_3 sum_k |RX_rk||t_k| + 2u (|RX t| + |tX|) (dot3 and the final addition of iso_mul)."""
    rs = np.random.RandomState(4)
    for i, w in enumerate(_angle_cases()[::3]):
        ax = rs.randn(3)
        ax /= np.linalg.norm(ax)
        X = np.eye(4)[:3].copy()
        R0, _ = rodrigues_exact(ax * rs.uniform(0, math.pi))
        X[:, :3] = np.array([[float(R0[r, c]) for c in range(3)] for r in range(3)])
        X[:, 3] = rs.uniform(-1e4, 1e4, 3) * (10.0 ** -(i % 4))
        t = rs.uniform(-2, 2, 3)
        dx = np.array([*t, *w])
        Xn = reg.solve_update(np.eye(N), -dx, X)
        R, th = rodrigues_exact(w)
        bar = rotation_bar(float(th))
        g3 = gamma(3)
        with mpmath.workprec(256):
            for r in range(3):
                for c in range(3):
                    ex = sum(mpmath.mpf(float(X[r, k])) * R[k, c] for k in range(3))
                    lim = sum(abs(X[r, k]) * (bar + g3 * abs(float(R[k, c]))) for k in range(3)) + U * abs(float(ex))
                    assert abs(mpmath.mpf(float(Xn[r, c])) - ex) <= lim * 1.01, (i, r, c)
                rt = sum(mpmath.mpf(float(X[r, k])) * mpmath.mpf(float(t[k])) for k in range(3))
                ex = rt + mpmath.mpf(float(X[r, 3]))
                lim = g3 * sum(abs(X[r, k] * t[k]) for k in range(3)) + 2 * U * (abs(float(rt)) + abs(X[r, 3]))
                assert abs(mpmath.mpf(float(Xn[r, 3])) - ex) <= lim * 1.01, (i, r)


# ====================================================================== GPU: keyframe weight
def _weight_cases(exact):
    hs = [H for _, H, _ in exact[::5]] + [H for _, H, _, _ in jacobian_cases() + golden_cases()]
    hs += [H for _, H, _, _, _ in tolerance_cases()] + [H for _, H, _ in special_zero_cases() + nan_inf_cases()]
    z = np.load(os.path.join(GOLD, "keyframe_weight_reference.npz"))
    hs += list(z["H"])
    rs = np.random.RandomState(12)
    for _ in range(40):  # general matrices: row exchanges at every step, signs of both kinds
        hs.append(rs.randn(N, N) * 10.0 ** rs.uniform(-3, 3))
    return hs


@pytest.mark.gpu
def test_weight_bitwise_with_the_oracle(exact, reg, oracle):
    for H in _weight_cases(exact):
        wd = reg.inv_det6(H)
        with np.errstate(all="ignore"):
            wo = oracle.inverse_determinant(H)
        assert bits_equal(np.array([wd]), np.array([wo])), (H, wd, wo)


@pytest.mark.gpu
def test_weight_against_the_exact_determinant(exact, reg):
    n = 0
    for H in [H for _, H, _ in exact[::5]] + [H for _, H, _, _ in jacobian_cases() + golden_cases()]:
        H = np.asarray(H, np.float64)
        d = det_bareiss(H)
        bar = _weight_bar(H) if d != 0 else None
        if bar is None:
            continue
        w = reg.inv_det6(H)
        assert math.isfinite(w) and (w > 0) == (d > 0), (w, float(d))
        assert abs(Fr(w) * d - 1) <= bar, (w, float(1 / d), float(bar))
        n += 1
    assert n >= 20


@pytest.mark.gpu
def test_weight_decisions_on_singular_H_follow_the_reference(reg):
    """keyframe_weight_reference.npz holds the reference's H.inverse().determinant() (make_weight_reference.py).
    Kind 0: exactly singular H whose partial-pivot LU meets its only zero pivot at the last step; where the running
    product is negative there, 1/det would be -inf and Pipeline's smallest-weight search would keep that frame.  The
    weight must make the same `<` decisions against finite weights as the reference's value.  Kind 2 (near-singular):
    both libraries return rounding noise; only finiteness is required of ours."""
    z = np.load(os.path.join(GOLD, "keyframe_weight_reference.npz"))
    finite = [-np.finfo(np.float64).max, -1.0, -1e-300, 0.0, 1e-300, 1.0, 1e300, np.finfo(np.float64).max]
    negative_zero_last = 0
    for H, kind, ref in zip(z["H"], z["kind"], z["ref_weight"]):
        w = reg.inv_det6(H)
        if kind == 2:
            assert math.isfinite(w), H
            continue
        if kind == 0:
            A = np.array(H)
            det = 1.0
            for k in range(N):  # the LU in inv_det6's order: the last pivot is exactly zero
                p = max(range(k, N), key=lambda i: (abs(A[i, k]), -i))
                if p != k:
                    A[[k, p]] = A[[p, k]]
                    det = -det
                det *= A[k, k]
                for i in range(k + 1, N):
                    A[i, k:] = A[i, k:] - (A[i, k] / A[k, k]) * A[k, k:]
            assert A[N - 1, N - 1] == 0.0 and all(A[k, k] != 0 for k in range(N - 1)), H
            negative_zero_last += bool(np.signbit(det))
        for f in finite:
            assert (w < f) == (ref < f) and (f < w) == (f < ref), (H, w, ref, f)
    assert negative_zero_last >= 6


# ====================================================================== GPU: the persistent kernel's solve is K3's
@pytest.fixture(scope="module")
def golden_regs(built, oracle):
    from mad_icp_b200 import FlatTree, Registrar, synth
    out = []
    c = synth.registration_case(K=2, beams=16, azimuths=512, seed=3)
    np.random.seed(42)
    cloud = synth.four_walls(points_per_wall=1000)
    g = np.load(os.path.join(GOLD, "four_walls_registration.npz"))
    walls = dict(scans=[cloud], kf_poses=[np.eye(4)], query=cloud.copy(), T_guess=g["T_guess"])
    for name, case in (("lidar_small", c), ("four_walls", walls)):
        r = Registrar(device=0, max_keyframes=len(case["scans"]))
        for k, (scan, P) in enumerate(zip(case["scans"], case["kf_poses"])):
            ft = FlatTree(scan)
            ft.apply_transform(P)
            r.put_keyframe(k, ft)
        q = FlatTree(case["query"])
        out.append((name, r, q.leaf_means(), case["T_guess"]))
    return out


@pytest.mark.gpu
def test_persistent_kernel_solve_is_k3(golden_regs):
    rank_deficient = 0
    for name, r, means, T in golden_regs:
        for moving, iters_list in ((means, (1, 3, 10)), (means[:2], (1, 4))):  # two moving leaves: rank <= 2 per kf
            r.set_moving(moving)
            for iters in iters_list:
                r.register_async(T, iters)
                out = r.register_fetch()
                tr = r.register_trace()
                assert tr.shape[0] == iters + 1
                assert bits_equal(out["X"], r.solve_update(out["H"], out["b"], tr[iters - 1])), (name, iters)
                assert bits_equal(out["X"], tr[iters]), (name, iters)
                assert bits_equal(np.array([out["weight"]]), np.array([r.inv_det6(out["H"])])), (name, iters)
                if moving is not means:
                    f = ldlt_factor(sym_lower(out["H"]))
                    rank_deficient += sum(d == 0 for d in factors(f)[1]) > 0 or np.linalg.matrix_rank(out["H"]) < N
    assert rank_deficient > 0
