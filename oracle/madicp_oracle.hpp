// =============================================================================
// oracle/madicp_oracle.hpp  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// Eigen-free CPU restatement of the reference's per-scan registration path
// (rvp-group/mad-icp @ v0.0.10).  Only tests/, __graft_entry__.smoke() and the
// cpu_baseline / `--impl reference` legs of bench.py may use it.  The product
// (mad_icp_b200/) never includes, links or calls anything in this directory.
//
// PARITY STATUS: the reference ships no tests/golden vectors, and it is built here
// without Eigen.  Two anchors exist:
//  (1) tests/test_reference_pin.py pins to the reference's OWN sources (from
//      a checkout of the reference, unmodified, compiled against oracle/eigen_standin; their
//      outputs are stored under tests/golden/) and requires this
//      restatement to equal them BIT FOR BIT (trees, searches, every GN round,
//      the streamed Pipeline).  Control flow, statement order and data handling
//      are therefore the reference's, verified.
//  (2) UNPINNED: the evaluation order inside Eigen's own operators.  This file
//      restates the three Eigen 3.4.0 routines the reference calls
//      (SelfAdjointEigenSolver<Matrix3d>::computeDirect, LDLT<Matrix6d>, fixed-size
//      coefficient products) from their published algorithm, the stand-in reuses
//      them, and where Eigen's floating-point evaluation order is not recoverable
//      from the reference tree the order is DEFINED here (see dot3) and the
//      product mirrors it.
//
// Each function cites the reference file:line it follows (paths relative to
// the reference's mad_icp/src).
//
// Build flags (oracle/Makefile): -O3 -fopenmp -std=c++17 -ffp-contract=off, no
// -march=native, no -ffast-math (reference: mad_icp/CMakeLists.txt:6-8,38-40).
// =============================================================================
#pragma once
#include <omp.h>

#include <cmath>
#include <cstddef>
#include <cstdint>
#include <cstring>
#include <limits>
#include <utility>
#include <vector>

namespace orc {

// ----------------------------------------------------------------------------
// Tiny fixed-size types standing in for Eigen::Vector3d / Matrix3d (column-major)
// ----------------------------------------------------------------------------
struct V3 {
  double v[3];
  double& operator[](int i) { return v[i]; }
  const double& operator[](int i) const { return v[i]; }
};
struct M3 {  // column-major like Eigen: (r,c) -> m[c*3+r]
  double m[9];
  double& operator()(int r, int c) { return m[c * 3 + r]; }
  const double& operator()(int r, int c) const { return m[c * 3 + r]; }
  V3 col(int c) const { return V3{{m[c * 3], m[c * 3 + 1], m[c * 3 + 2]}}; }
  void setCol(int c, const V3& x) {
    m[c * 3] = x[0];
    m[c * 3 + 1] = x[1];
    m[c * 3 + 2] = x[2];
  }
};
struct Iso3 {  // Eigen::Isometry3d: linear() + translation()
  M3 R;
  V3 t;
};
struct M6 {  // column-major 6x6
  double m[36];
  double& operator()(int r, int c) { return m[c * 6 + r]; }
  const double& operator()(int r, int c) const { return m[c * 6 + r]; }
};
struct V6 {
  double v[6];
};

inline V3 sub(const V3& a, const V3& b) { return V3{{a[0] - b[0], a[1] - b[1], a[2] - b[2]}}; }
inline V3 add(const V3& a, const V3& b) { return V3{{a[0] + b[0], a[1] + b[1], a[2] + b[2]}}; }
// DEFINED ORDER for every 3-term coefficient sum (Eigen's redux order for a
// 3-vector is not recoverable here): ((a0*b0 + a1*b1) + a2*b2), no FMA.
inline double dot3(const V3& a, const V3& b) { return (a[0] * b[0] + a[1] * b[1]) + a[2] * b[2]; }
inline double norm3(const V3& a) { return std::sqrt(dot3(a, a)); }
inline V3 cross3(const V3& a, const V3& b) {
  return V3{{a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]}};
}
inline V3 mulMV(const M3& A, const V3& x) {  // rows of A dotted with x
  V3 r;
  for (int i = 0; i < 3; ++i) r[i] = (A(i, 0) * x[0] + A(i, 1) * x[1]) + A(i, 2) * x[2];
  return r;
}
inline M3 mulMM(const M3& A, const M3& B) {
  M3 C;
  for (int j = 0; j < 3; ++j)
    for (int i = 0; i < 3; ++i) C(i, j) = (A(i, 0) * B(0, j) + A(i, 1) * B(1, j)) + A(i, 2) * B(2, j);
  return C;
}
inline V3 isoApply(const Iso3& X, const V3& p) { return add(mulMV(X.R, p), X.t); }  // linear*p + translation
inline Iso3 isoMul(const Iso3& A, const Iso3& B) {
  Iso3 C;
  C.R = mulMM(A.R, B.R);
  C.t = add(mulMV(A.R, B.t), A.t);
  return C;
}
inline M3 identity3() {
  M3 I;
  std::memset(I.m, 0, sizeof(I.m));
  I(0, 0) = I(1, 1) = I(2, 2) = 1.0;
  return I;
}

// ----------------------------------------------------------------------------
// tools/lie_algebra.h:33-37  skew ; :39-52  expMapSO3
// ----------------------------------------------------------------------------
inline M3 skew(const V3& v) {
  M3 S;
  S(0, 0) = 0.0;   S(0, 1) = -v[2]; S(0, 2) = v[1];
  S(1, 0) = v[2];  S(1, 1) = 0.0;   S(1, 2) = -v[0];
  S(2, 0) = -v[1]; S(2, 1) = v[0];  S(2, 2) = 0.0;
  return S;
}
inline M3 expMapSO3(const V3& omega) {
  M3 R;
  const double theta_square = dot3(omega, omega);
  const double theta = std::sqrt(theta_square);
  const M3 W = skew(omega);
  M3 K;
  for (int i = 0; i < 9; ++i) K.m[i] = W.m[i] / theta;  // Inf/NaN when theta==0, unused then
  const M3 I = identity3();
  if (theta_square < 1e-8) {
    for (int i = 0; i < 9; ++i) R.m[i] = I.m[i] + W.m[i];
  } else {
    const double one_minus_cos = 2.0 * std::sin(theta / 2.0) * std::sin(theta / 2.0);
    const double s = std::sin(theta);
    M3 oK;
    for (int i = 0; i < 9; ++i) oK.m[i] = one_minus_cos * K.m[i];
    const M3 oKK = mulMM(oK, K);
    for (int i = 0; i < 9; ++i) R.m[i] = (I.m[i] + s * K.m[i]) + oKK.m[i];
  }
  return R;
}

// ----------------------------------------------------------------------------
// Eigen 3.4.0 SelfAdjointEigenSolver<Matrix3d>::computeDirect, restated from the
// published algorithm (closed-form trigonometric roots + cross-product kernel
// extraction).  Called at tools/mad_tree.cpp:59-61.  Only eigenvectors are
// consumed by the reference.  Eigenvalues ascending: col(0)=normal, col(2)=split.
// ----------------------------------------------------------------------------
inline void eig3_roots(const M3& m, double roots[3]) {
  const double s_inv3 = 1.0 / 3.0;
  const double s_sqrt3 = std::sqrt(3.0);
  const double c0 = m(0, 0) * m(1, 1) * m(2, 2) + 2.0 * m(1, 0) * m(2, 0) * m(2, 1) - m(0, 0) * m(2, 1) * m(2, 1) -
                    m(1, 1) * m(2, 0) * m(2, 0) - m(2, 2) * m(1, 0) * m(1, 0);
  const double c1 = m(0, 0) * m(1, 1) - m(1, 0) * m(1, 0) + m(0, 0) * m(2, 2) - m(2, 0) * m(2, 0) + m(1, 1) * m(2, 2) -
                    m(2, 1) * m(2, 1);
  const double c2 = m(0, 0) + m(1, 1) + m(2, 2);
  const double c2_over_3 = c2 * s_inv3;
  double a_over_3 = (c2 * c2_over_3 - c1) * s_inv3;
  a_over_3 = (a_over_3 < 0.0) ? 0.0 : a_over_3;  // numext::maxi(a,0): returns a unless a<0 (NaN stays NaN)
  const double half_b = 0.5 * (c0 + c2_over_3 * (2.0 * c2_over_3 * c2_over_3 - c1));
  double q = a_over_3 * a_over_3 * a_over_3 - half_b * half_b;
  q = (q < 0.0) ? 0.0 : q;
  const double rho = std::sqrt(a_over_3);
  const double theta = std::atan2(std::sqrt(q), half_b) * s_inv3;
  const double cos_theta = std::cos(theta);
  const double sin_theta = std::sin(theta);
  roots[0] = c2_over_3 - rho * (cos_theta + s_sqrt3 * sin_theta);
  roots[1] = c2_over_3 - rho * (cos_theta - s_sqrt3 * sin_theta);
  roots[2] = c2_over_3 + 2.0 * rho * cos_theta;
}
inline void eig3_extract_kernel(const M3& mat, V3& res, V3& representative) {
  // column of the largest |diagonal| entry (first maximum wins)
  int i0 = 0;
  double best = std::fabs(mat(0, 0));
  for (int i = 1; i < 3; ++i) {
    const double a = std::fabs(mat(i, i));
    if (a > best) {
      best = a;
      i0 = i;
    }
  }
  representative = mat.col(i0);
  const V3 c0 = cross3(representative, mat.col((i0 + 1) % 3));
  const V3 c1 = cross3(representative, mat.col((i0 + 2) % 3));
  const double n0 = dot3(c0, c0);
  const double n1 = dot3(c1, c1);
  if (n0 > n1) {
    const double d = std::sqrt(n0);
    res = V3{{c0[0] / d, c0[1] / d, c0[2] / d}};
  } else {
    const double d = std::sqrt(n1);
    res = V3{{c1[0] / d, c1[1] / d, c1[2] / d}};
  }
}
inline void eig3_computeDirect(const M3& mat, M3& eivecs, double eivals[3]) {
  const double shift = (mat(0, 0) + mat(1, 1) + mat(2, 2)) / 3.0;
  M3 scaledMat;  // selfadjointView<Lower>
  for (int c = 0; c < 3; ++c)
    for (int r = 0; r < 3; ++r) scaledMat(r, c) = (r >= c) ? mat(r, c) : mat(c, r);
  for (int i = 0; i < 3; ++i) scaledMat(i, i) -= shift;
  double scale = std::fabs(scaledMat.m[0]);
  for (int i = 1; i < 9; ++i) {
    const double a = std::fabs(scaledMat.m[i]);
    if (a > scale) scale = a;
  }
  if (scale > 0.0)
    for (int i = 0; i < 9; ++i) scaledMat.m[i] /= scale;
  eig3_roots(scaledMat, eivals);
  const double eps = std::numeric_limits<double>::epsilon();
  if ((eivals[2] - eivals[0]) <= eps) {
    eivecs = identity3();
  } else {
    M3 tmp = scaledMat;
    double d0 = eivals[2] - eivals[1];
    double d1 = eivals[1] - eivals[0];
    int k = 0, l = 2;
    if (d0 > d1) {
      std::swap(k, l);
      d0 = d1;
    }
    V3 vk, vl;
    {
      for (int i = 0; i < 3; ++i) tmp(i, i) -= eivals[k];
      eig3_extract_kernel(tmp, vk, vl);
    }
    if (d0 <= 2.0 * eps * d1) {
      const double d = dot3(vk, vl);
      for (int i = 0; i < 3; ++i) vl[i] -= d * vl[i];
      const double n = norm3(vl);
      for (int i = 0; i < 3; ++i) vl[i] /= n;
    } else {
      tmp = scaledMat;
      for (int i = 0; i < 3; ++i) tmp(i, i) -= eivals[l];
      V3 dummy;
      eig3_extract_kernel(tmp, vl, dummy);
    }
    eivecs.setCol(k, vk);
    eivecs.setCol(l, vl);
    V3 mid = cross3(eivecs.col(2), eivecs.col(0));
    const double n = norm3(mid);
    for (int i = 0; i < 3; ++i) mid[i] /= n;
    eivecs.setCol(1, mid);
  }
  for (int i = 0; i < 3; ++i) eivals[i] = eivals[i] * scale + shift;
}

// ----------------------------------------------------------------------------
// Eigen 3.4.0 LDLT<Matrix6d>::compute + solve, restated (lower storage, diagonal
// pivoting, pseudo-inverse of D with tolerance = numeric_limits<double>::min()).
// Called at odometry/mad_icp.cpp:111.
// ----------------------------------------------------------------------------
inline void ldlt6_solve(const M6& Hin, const V6& rhs, V6& x) {
  const int n = 6;
  double A[6][6];
  for (int r = 0; r < n; ++r)
    for (int c = 0; c < n; ++c) A[r][c] = Hin(r, c);  // only lower part is read below
  int tr[6];
  for (int k = 0; k < n; ++k) {
    int big = k;
    double bv = std::fabs(A[k][k]);
    for (int i = k + 1; i < n; ++i) {
      const double a = std::fabs(A[i][i]);
      if (a > bv) {
        bv = a;
        big = i;
      }
    }
    tr[k] = big;
    if (k != big) {
      for (int j = 0; j < k; ++j) std::swap(A[k][j], A[big][j]);
      for (int i = big + 1; i < n; ++i) std::swap(A[i][k], A[i][big]);
      std::swap(A[k][k], A[big][big]);
      for (int i = k + 1; i < big; ++i) std::swap(A[i][k], A[big][i]);
    }
    const int rs = n - k - 1;
    if (k > 0) {
      double temp[6];
      for (int j = 0; j < k; ++j) temp[j] = A[j][j] * A[k][j];
      double s = 0.0;
      for (int j = 0; j < k; ++j) s += A[k][j] * temp[j];
      A[k][k] -= s;
      for (int i = k + 1; i < n; ++i) {
        double s2 = 0.0;
        for (int j = 0; j < k; ++j) s2 += A[i][j] * temp[j];
        A[i][k] -= s2;
      }
    }
    const double akk = A[k][k];
    const bool pivot_is_valid = std::fabs(akk) > 0.0;
    if (k == 0 && !pivot_is_valid) {
      for (int j = 0; j < n; ++j) tr[j] = j;
      break;
    }
    if (rs > 0 && pivot_is_valid)
      for (int i = k + 1; i < n; ++i) A[i][k] /= akk;
  }
  double y[6];
  for (int i = 0; i < n; ++i) y[i] = rhs.v[i];
  for (int k = 0; k < n; ++k)
    if (tr[k] != k) std::swap(y[k], y[tr[k]]);
  for (int i = 0; i < n; ++i)  // L y = P b (unit lower)
    for (int j = 0; j < i; ++j) y[i] -= A[i][j] * y[j];
  const double tol = std::numeric_limits<double>::min();
  for (int i = 0; i < n; ++i) {
    if (std::fabs(A[i][i]) > tol)
      y[i] /= A[i][i];
    else
      y[i] = 0.0;
  }
  for (int i = n - 1; i >= 0; --i)  // L^T x = y
    for (int j = i + 1; j < n; ++j) y[i] -= A[j][i] * y[j];
  for (int k = n - 1; k >= 0; --k)
    if (tr[k] != k) std::swap(y[k], y[tr[k]]);
  for (int i = 0; i < n; ++i) x.v[i] = y[i];
}

// ----------------------------------------------------------------------------
// tools/mad_tree.h:47-102  node type.  Field order follows :91-98 so the heap
// object is 152 bytes and the CPU baseline has the reference's memory behaviour.
// ----------------------------------------------------------------------------
struct Tree;
using Cloud = std::vector<V3>;
using LeafList = std::vector<Tree*>;

struct Tree {
  int num_points_;
  bool matched_;
  Tree* left_ = nullptr;
  Tree* right_ = nullptr;
  Tree* parent_ = nullptr;
  V3 mean_;
  V3 bbox_;
  M3 eigenvectors_;

  Tree(Cloud* vec, size_t begin, size_t end, double b_max, double b_min, int level, int max_parallel_level, Tree* parent,
       Tree* plane_predecessor) {
    matched_ = false;
    build(vec, begin, end, b_max, b_min, level, max_parallel_level, parent, plane_predecessor);
  }
  ~Tree() {
    if (left_) delete left_;
    if (right_) delete right_;
  }

  // tools/utils.h:55-73
  static int computeMeanAndCovariance(V3& mean, M3& cov, const Cloud& c, size_t begin, size_t end) {
    mean = V3{{0, 0, 0}};
    std::memset(cov.m, 0, sizeof(cov.m));
    int k = 0;
    for (size_t it = begin; it != end; ++it) {
      const V3& v = c[it];
      for (int i = 0; i < 3; ++i) mean[i] += v[i];
      for (int cc = 0; cc < 3; ++cc)
        for (int r = 0; r < 3; ++r) cov(r, cc) += v[r] * v[cc];
      ++k;
    }
    const double inv = 1. / k;
    for (int i = 0; i < 3; ++i) mean[i] *= inv;
    for (int i = 0; i < 9; ++i) cov.m[i] *= inv;
    for (int cc = 0; cc < 3; ++cc)
      for (int r = 0; r < 3; ++r) cov(r, cc) -= mean[r] * mean[cc];
    const double f = double(k) / double(k - 1);
    for (int i = 0; i < 9; ++i) cov.m[i] *= f;
    return k;
  }
  // tools/utils.h:76-97 ; R = eigenvectors^T so v(i) = col(i) . (p - center)
  static int computeBoundingBox(V3& b_max, const V3& center, const M3& eivecs, const Cloud& c, size_t begin, size_t end) {
    int k = 0;
    V3 neg{{0, 0, 0}}, pos{{0, 0, 0}};
    for (size_t it = begin; it != end; ++it) {
      const V3 d = sub(c[it], center);
      for (int i = 0; i < 3; ++i) {
        const double vi = dot3(eivecs.col(i), d);
        neg[i] = (vi < neg[i]) ? vi : neg[i];  // std::min(a,b) = (b<a)?b:a  -> NaN ignored
        pos[i] = (pos[i] < vi) ? vi : pos[i];  // std::max(a,b) = (a<b)?b:a
      }
      ++k;
    }
    b_max = sub(pos, neg);
    return k;
  }

  // tools/mad_tree.cpp:47-130 (std::async top levels omitted: result is independent of it)
  void build(Cloud* vec, size_t begin, size_t end, double b_max, double b_min, int level, int max_parallel_level,
             Tree* parent, Tree* plane_predecessor) {
    parent_ = parent;
    M3 cov;
    computeMeanAndCovariance(mean_, cov, *vec, begin, end);
    double evals[3];
    eig3_computeDirect(cov, eigenvectors_, evals);
    num_points_ = computeBoundingBox(bbox_, mean_, eigenvectors_, *vec, begin, end);

    if (bbox_[2] < b_max) {
      if (plane_predecessor) {
        eigenvectors_.setCol(0, plane_predecessor->eigenvectors_.col(0));
      } else {
        if (num_points_ < 3) {
          Tree* node = this;
          while (node->parent_ && node->num_points_ < 3) node = node->parent_;
          eigenvectors_.setCol(0, node->eigenvectors_.col(0));
        }
      }
      V3& nearest_point = (*vec)[begin];  // reference writes through this alias (mad_tree.cpp:76,82)
      double shortest_dist = std::numeric_limits<double>::max();
      for (size_t it = begin; it != end; ++it) {
        const V3& v = (*vec)[it];
        const double dist = norm3(sub(v, mean_));
        if (dist < shortest_dist) {
          nearest_point = v;
          shortest_dist = dist;
        }
      }
      mean_ = nearest_point;
      return;
    }
    if (!plane_predecessor) {
      if (bbox_[0] < b_min) plane_predecessor = this;
    }
    const V3 n = eigenvectors_.col(2);
    // tools/utils.h:38-52 split
    size_t lower = begin, upper = end;
    Cloud& c = *vec;
    while (lower != upper) {
      if (dot3(sub(c[lower], mean_), n) < double(0)) {
        ++lower;
      } else {
        std::swap(c[lower], c[upper - 1]);
        --upper;
      }
    }
    const size_t middle = upper;
    left_ = new Tree(vec, begin, middle, b_max, b_min, level + 1, max_parallel_level, this, plane_predecessor);
    right_ = new Tree(vec, middle, end, b_max, b_min, level + 1, max_parallel_level, this, plane_predecessor);
  }

  // tools/mad_tree.cpp:144-152
  const Tree* bestMatchingLeafFast(const V3& query) const {
    const Tree* node = this;
    while (node->left_ || node->right_) {
      const V3 n = node->eigenvectors_.col(2);
      node = (dot3(sub(query, node->mean_), n) < double(0)) ? node->left_ : node->right_;
    }
    return node;
  }
  // tools/mad_tree.cpp:154-163
  void getLeafs(LeafList& out) {
    if (!left_ && !right_) {
      out.push_back(this);
      return;
    }
    if (left_) left_->getLeafs(out);
    if (right_) right_->getLeafs(out);
  }
  // tools/mad_tree.cpp:165-172
  void applyTransform(const M3& r, const V3& t) {
    mean_ = add(mulMV(r, mean_), t);
    eigenvectors_ = mulMM(r, eigenvectors_);
    if (left_) left_->applyTransform(r, t);
    if (right_) right_->applyTransform(r, t);
  }
};
static_assert(sizeof(Tree) == 152, "node must match the reference's 152-byte heap object");

// ----------------------------------------------------------------------------
// odometry/mad_icp.{h,cpp}  MADicp
// ----------------------------------------------------------------------------
struct MADicp {
  Iso3 X_;
  M6 H_adder_;
  V6 b_adder_;
  LeafList moving_leaves_;
  std::vector<M6> H_adders_;
  std::vector<V6> b_adders_;
  double rho_ker_, min_ball_, b_ratio_;
  int num_threads_;

  // mad_icp.cpp:31-39
  MADicp(double min_ball, double rho_ker, double b_ratio, int num_threads)
      : rho_ker_(std::sqrt(rho_ker)), min_ball_(min_ball), b_ratio_(b_ratio), num_threads_(num_threads) {
    X_.R = identity3();
    X_.t = V3{{0, 0, 0}};
    std::memset(&H_adder_, 0, sizeof(H_adder_));
    std::memset(&b_adder_, 0, sizeof(b_adder_));
    H_adders_.resize(num_threads);
    b_adders_.resize(num_threads);
  }
  // mad_icp.cpp:41-49
  void resetAdders() {
    std::memset(&H_adder_, 0, sizeof(H_adder_));
    std::memset(&b_adder_, 0, sizeof(b_adder_));
    for (int i = 0; i < num_threads_; ++i) {
      std::memset(&H_adders_[i], 0, sizeof(M6));
      std::memset(&b_adders_[i], 0, sizeof(V6));
    }
  }
  void setMoving(const LeafList& l) { moving_leaves_ = l; }  // :51-53
  void init(const Iso3& X) { X_ = X; }                        // :55-57

  // mad_icp.cpp:59-72
  void errorAndJacobian(double& e, double J[6], const Tree& fixed, const Tree& moving, const V3& moving_transformed) const {
    const V3& fixed_point = fixed.mean_;
    const V3 fixed_normal = fixed.eigenvectors_.col(0);
    const V3& moving_point = moving.mean_;
    const M3& R = X_.R;
    e = dot3(sub(moving_transformed, fixed_point), fixed_normal);
    for (int j = 0; j < 3; ++j) J[j] = (fixed_normal[0] * R(0, j) + fixed_normal[1] * R(1, j)) + fixed_normal[2] * R(2, j);
    const M3 S = skew(moving_point);
    const double nJ[3] = {-J[0], -J[1], -J[2]};
    for (int j = 0; j < 3; ++j) J[3 + j] = (nJ[0] * S(0, j) + nJ[1] * S(1, j)) + nJ[2] * S(2, j);
  }

  // mad_icp.cpp:74-103.  `idx_out` (nullable) is instrumentation: it records the
  // address of the matched leaf for every moving leaf, BEFORE the gate.
  void update(const Tree* fixed_tree, const Tree** idx_out = nullptr) {
    const int thread_id = omp_get_thread_num();
    size_t qi = 0;
    for (auto& moving : moving_leaves_) {
      const V3 ml = isoApply(X_, moving->mean_);
      const Tree* f = fixed_tree->bestMatchingLeafFast(ml);
      if (idx_out) idx_out[qi] = f;
      ++qi;
      const double src_ball = min_ball_ + b_ratio_ * norm3(moving->mean_);
      if (norm3(sub(ml, f->mean_)) > src_ball) continue;
      moving->matched_ = true;
      double J[6];
      double e;
      errorAndJacobian(e, J, *f, *moving, ml);
      double scale = 1.;
      const double chi = std::fabs(e);  // SURVEY F10: double abs in the x86-64 reference build
      if (chi > rho_ker_) scale = rho_ker_ / chi;
      const double w = 1. - f->bbox_[0] / min_ball_;
      scale *= w * w;
      M6& H = H_adders_[thread_id];
      V6& b = b_adders_[thread_id];
      double sJ[6];
      for (int i = 0; i < 6; ++i) sJ[i] = scale * J[i];
      for (int c = 0; c < 6; ++c)
        for (int r = 0; r < 6; ++r) H(r, c) += sJ[r] * J[c];
      for (int r = 0; r < 6; ++r) b.v[r] += sJ[r] * e;
    }
  }

  // mad_icp.cpp:105-117
  void updateState() {
    for (int i = 0; i < num_threads_; ++i) {
      for (int j = 0; j < 36; ++j) H_adder_.m[j] += H_adders_[i].m[j];
      for (int j = 0; j < 6; ++j) b_adder_.v[j] += b_adders_[i].v[j];
    }
    V6 nb, dx;
    for (int j = 0; j < 6; ++j) nb.v[j] = -b_adder_.v[j];
    ldlt6_solve(H_adder_, nb, dx);
    Iso3 dX;
    dX.R = expMapSO3(V3{{dx.v[3], dx.v[4], dx.v[5]}});
    dX.t = V3{{dx.v[0], dx.v[1], dx.v[2]}};
    X_ = isoMul(X_, dX);
  }
};

// ----------------------------------------------------------------------------
// ICP driver loop: odometry/pipeline.cpp:166-193 (OpenMP parallel-for over the
// keyframes, matched_ cleared before the last iteration) which for one keyframe
// and one thread is pybind/tools/mad_icp_wrapper.h:72-81.
// Optional per-iteration recording (poses before each iteration, H, b, matched
// leaf per (keyframe, moving leaf)) is instrumentation for the parity tests.
// ----------------------------------------------------------------------------
struct IcpRecord {
  std::vector<Iso3> X_before;                    // iters entries
  std::vector<M6> H;                             // iters entries (H_adder_ after updateState)
  std::vector<V6> b;                             // iters
  std::vector<std::vector<const Tree*>> matches; // iters x (K*L)
};

inline void icp_loop(MADicp& icp, const std::vector<Tree*>& keyframes, LeafList& moving, int iters, int num_threads,
                     IcpRecord* rec, bool record_matches) {
  const int K = (int) keyframes.size();
  const size_t L = moving.size();
  omp_set_num_threads(num_threads);
  for (int it = 0; it < iters; ++it) {
    if (it == iters - 1)
      for (Tree* l : moving) l->matched_ = false;
    icp.resetAdders();
    if (rec) rec->X_before.push_back(icp.X_);
    const Tree** mrow = nullptr;
    if (rec && record_matches) {
      rec->matches.emplace_back(size_t(K) * L);
      mrow = rec->matches.back().data();
    }
#pragma omp parallel for
    for (int k = 0; k < K; ++k) { icp.update(keyframes[k], mrow ? mrow + size_t(k) * L : nullptr); }
    icp.updateState();
    if (rec) {
      rec->H.push_back(icp.H_adder_);
      rec->b.push_back(icp.b_adder_);
    }
  }
}

}  // namespace orc
