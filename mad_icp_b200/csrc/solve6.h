// solve6.h -- Gauss-Newton state update shared by host and device:
//   dx = H.ldlt().solve(-b);  dX = (expMapSO3(dx[3:6]), dx[0:3]);  X = X * dX
// (reference: odometry/mad_icp.cpp:105-117, tools/lie_algebra.h:33-52).
//
// The factorisation is the pivoted lower LDL^T that Eigen 3.4's LDLT<Matrix6d> performs (largest
// |diagonal| first, pseudo-inverse of D in the solve so a rank-deficient or all-zero H gives dx = 0
// on the null space instead of NaN).  That algorithm is left-looking: column k is only updated when
// it becomes the pivot column, so the pivot search at step k looks at diagonal entries that are
// still the ORIGINAL ones.  The whole pivot order is therefore a function of diag(H) alone, and the
// routine below (1) derives the permutation from the diagonal, (2) gathers the permuted lower
// triangle with run-time indices from memory once, (3) runs the same left-looking elimination
// un-pivoted with compile-time indices only.  On the device that keeps the working set in
// registers; the update sits on the critical path between two GN rounds (one thread, nothing to
// overlap with), and a pointer-indexed version costs ~25 us per round.
// tests/test_gpu_update.py checks these claims against an exact rational LDL^T written from Eigen's algorithm: all
// 720 pivot orders, every rank, ties of the largest diagonal that change the answer, the DBL_MIN cut-off of the
// pseudo-inverse, and an upper triangle that is NaN or differs from the lower one.
#pragma once
#include <float.h>

#include "arith.h"

namespace madicp {

#if defined(__CUDACC__)
#define MADICP_HD_COLD static __host__ __device__ __noinline__
#else
#define MADICP_HD_COLD inline
#endif

// The solve when the first pivot is 0 (the whole diagonal is zero, NaN entries aside) or NaN (H[0][0] is NaN, which
// no other entry beats).  Eigen stops factoring there and solves with the untouched lower triangle as L and D, in the
// original order: 0 for a finite H, and NaN where Eigen's own solve meets one.  Out of line, so that the persistent
// kernel does not carry its registers for a case that finite sums of J^T J never reach.
MADICP_HD_COLD void ldlt6_solve_neg_unfactored(const double* H, int ld, const double* b, double* x) {
  for (int i = 0; i < 6; ++i) {
    double v = -b[i];
    for (int j = 0; j < i; ++j) v -= H[i * ld + j] * x[j];
    x[i] = v;
  }
  for (int i = 0; i < 6; ++i) x[i] = (fabs(H[i * ld + i]) > DBL_MIN) ? x[i] / H[i * ld + i] : 0.0;
  for (int i = 5; i >= 0; --i)
    for (int j = i + 1; j < 6; ++j) x[i] -= H[j * ld + i] * x[j];
}

// H: 6x6 with row stride `ld` (H[r*ld+c]); only the lower triangle (r >= c) is read.  x = solve(-b).
MADICP_HD void ldlt6_solve_neg(const double* H, int ld, const double* b, double* x) {
  // (1) pivot order from the diagonal: selection with "first maximum wins", as sequential swaps
  double dg[6];
  int idx[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
    dg[i] = fabs(H[i * ld + i]);
    idx[i] = i;
  }
#pragma unroll
  for (int k = 0; k < 5; ++k) {
    int p = k;
    double best = dg[k];
#pragma unroll
    for (int i = k + 1; i < 6; ++i)
      if (dg[i] > best) {
        best = dg[i];
        p = i;
      }
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {
      const bool sw = (p == i);
      const double u = dg[k], w = dg[i];
      dg[k] = sw ? w : u;
      dg[i] = sw ? u : w;
      const int a = idx[k], c = idx[i];
      idx[k] = sw ? c : a;
      idx[i] = sw ? a : c;
    }
  }
  if (!(dg[0] > 0.0)) {
    ldlt6_solve_neg_unfactored(H, ld, b, x);
    return;
  }
  // (2) permuted lower triangle (entry (i,j) comes from the original LOWER entry of rows idx[i], idx[j])
  double A[6][6];
  double y[6];
#pragma unroll
  for (int i = 0; i < 6; ++i) {
#pragma unroll
    for (int j = 0; j <= i; ++j) {
      const int r = idx[i] > idx[j] ? idx[i] : idx[j];
      const int c = idx[i] > idx[j] ? idx[j] : idx[i];
      A[i][j] = H[r * ld + c];
    }
    y[i] = -b[idx[i]];
  }
  // (3) left-looking LDL^T, static indices
  double inv[6];
  bool keep[6];
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    if (k > 0) {
      double w[6];
#pragma unroll
      for (int j = 0; j < k; ++j) w[j] = A[j][j] * A[k][j];
      double s = 0.0;
#pragma unroll
      for (int j = 0; j < k; ++j) s += A[k][j] * w[j];
      A[k][k] -= s;
#pragma unroll
      for (int i = k + 1; i < 6; ++i) {
        double s2 = 0.0;
#pragma unroll
        for (int j = 0; j < k; ++j) s2 += A[i][j] * w[j];
        A[i][k] -= s2;
      }
    }
    const double d = A[k][k];
    // one reciprocal per pivot instead of a division per entry (Eigen divides; the quotients differ by
    // <= 1 ulp, far inside the pose tolerance, and a software DDIV is ~25 instructions on the serial path)
    keep[k] = fabs(d) > DBL_MIN;
    inv[k] = keep[k] ? 1.0 / d : 0.0;
    if (keep[k]) {
#pragma unroll
      for (int i = k + 1; i < 6; ++i) A[i][k] *= inv[k];
    } else if (fabs(d) > 0.0) {
      // a subnormal pivot: its reciprocal may overflow, and 0 * inf would put NaN where Eigen's 0 / d puts 0
#pragma unroll
      for (int i = k + 1; i < 6; ++i) A[i][k] /= d;
    }
  }
#pragma unroll
  for (int i = 0; i < 6; ++i)
#pragma unroll
    for (int j = 0; j < i; ++j) y[i] -= A[i][j] * y[j];
#pragma unroll
  for (int i = 0; i < 6; ++i) y[i] = keep[i] ? y[i] * inv[i] : 0.0;  // pseudo-inverse of D: Eigen sets these to 0
#pragma unroll
  for (int i = 5; i >= 0; --i)
#pragma unroll
    for (int j = i + 1; j < 6; ++j) y[i] -= A[j][i] * y[j];
#pragma unroll
  for (int i = 0; i < 6; ++i) x[idx[i]] = y[i];
}

// det(H^-1) as 1 / det(H) by partial-pivot LU (reference: odometry/pipeline.cpp:223 computes
// H_adder_.inverse().determinant(); the C++ facade uses the same form).  H row-major 6x6, stride ld.
MADICP_HD double inv_det6(const double* H, int ld) {
  // static indices only (the row exchange is a chain of selects): on the device the 6x6 stays in registers -- indexed
  // at run time it lived in local memory and the routine cost 4.6k cycles at the end of every registration
  double A[6][6];
#pragma unroll
  for (int r = 0; r < 6; ++r)
#pragma unroll
    for (int c = 0; c < 6; ++c) A[r][c] = H[r * ld + c];
  double det = 1.0;
#pragma unroll
  for (int k = 0; k < 6; ++k) {
    int p = k;
    double best = fabs(A[k][k]);
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {  // first maximum of |A[i][k]|, i >= k
      const double a = fabs(A[i][k]);
      if (a > best) {
        best = a;
        p = i;
      }
    }
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {  // rows k <-> p (columns left of k are never read again)
      const bool sw = (p == i);
#pragma unroll
      for (int c = k; c < 6; ++c) {
        const double u = A[k][c], w = A[i][c];
        A[k][c] = sw ? w : u;
        A[i][c] = sw ? u : w;
      }
    }
    if (p != k) det = -det;
    det = mul_(det, A[k][k]);
#pragma unroll
    for (int i = k + 1; i < 6; ++i) {
      const double f = A[i][k] / A[k][k];
#pragma unroll
      for (int c = k; c < 6; ++c) A[i][c] = sub_(A[i][c], mul_(f, A[k][c]));
    }
  }
  // An exactly zero pivot before the last one makes the rows below it 0/0, so det is already NaN.  A zero last pivot
  // leaves det = +-0, and 1/det would be +-inf: -inf is below every finite weight, and Pipeline would keep that
  // singular frame as a keyframe.  The reference's H.inverse() divides by that pivot, and the determinant of the
  // result is NaN, which never wins the smallest-weight search: return the same.
  return (A[5][5] == 0.0) ? NAN : 1.0 / det;
}

// Rodrigues with the reference's small-angle branch (theta^2 < 1e-8 -> I + [w]x). R row-major 3x3.
MADICP_HD void expmap_so3(double wx, double wy, double wz, double* R) {
  const double th2 = dot3(wx, wy, wz, wx, wy, wz);
  const double W[9] = {0.0, -wz, wy, wz, 0.0, -wx, -wy, wx, 0.0};
  if (th2 < 1e-8) {
#pragma unroll
    for (int i = 0; i < 9; ++i) R[i] = ((i % 4) == 0 ? 1.0 : 0.0) + W[i];
    return;
  }
  const double th = sqrt(th2);
  const double inv_th = 1.0 / th;
  double K[9], oK[9];
#pragma unroll
  for (int i = 0; i < 9; ++i) K[i] = W[i] * inv_th;
  const double hs = sin(th / 2.0);
  const double omc = 2.0 * hs * hs;
  const double s = sin(th);
#pragma unroll
  for (int i = 0; i < 9; ++i) oK[i] = omc * K[i];
#pragma unroll
  for (int r = 0; r < 3; ++r)
#pragma unroll
    for (int c = 0; c < 3; ++c) {
      const double kk = dot3(oK[r * 3], oK[r * 3 + 1], oK[r * 3 + 2], K[c], K[3 + c], K[6 + c]);
      R[r * 3 + c] = (((r == c) ? 1.0 : 0.0) + s * K[r * 3 + c]) + kk;
    }
}

// Xn (row-major 3x4) = X * [exp(w) | t] with dx = [t, w] solved from (H, b); H has row stride ld.
MADICP_HD void gn_update_pose(const double* H, int ld, const double* b, const double* X, double* Xn) {
  double dx[6];
  ldlt6_solve_neg(H, ld, b, dx);
  double dR[9], dX[12];
  expmap_so3(dx[3], dx[4], dx[5], dR);
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) dX[r * 4 + c] = dR[r * 3 + c];
    dX[r * 4 + 3] = dx[r];
  }
  iso_mul(X, dX, Xn);
}

}  // namespace madicp
