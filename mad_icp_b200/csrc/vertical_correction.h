// vertical_correction.h -- KITTI's vertical-angle correction as ONE restatement shared by host C++ and sm_90a device
// code, bit for bit with the reader it replaces (apps/utils/kitti_reader.py:72-79, applied after the range mask at
// :90-91):
//   rv = np.cross(points, [0., 0., 1.]); rvn = rv / np.linalg.norm(rv, axis=1)[:, None]
//   points = Rotation.from_rotvec(theta * rvn).apply(points)          (theta = np.radians(0.205) in the reader)
// Spelled out (c = the float64 of the point's field values; every operation rounded, left to right, no FMA):
//   c0 = y*1 - z*0,  c1 = z*0 - x*1,  c2 = x*0 - y*0     (np.cross with a float64 [0,0,1]: the *0 / *1 terms decide
//                                                        the signs of zeros and where inf / NaN go)
//   n = sqrt((c0*c0 + c1*c1) + c2*c2),  r_i = theta * (c_i / n),  a = sqrt((r0*r0 + r1*r1) + r2*r2)
//   s = a <= 1e-3 ? (0.5 - a2/48) + a2*a2/3840 (a2 = a*a) : sin(a/2)/a,  w = cos(a/2)     (scipy's from_rotvec)
//   q = (s*r0, s*r1, s*r2, w), m = the rotation matrix of q (scipy's order below),
//   out_r = ((0 + m_r0*x) + m_r2*z) + m_r1*y
// The last line is scipy's order: its sum starts from +0 (which turns a -0 result into +0) and takes the columns in
// the order 0, 2, 1; (m_r0*x + m_r1*y) + m_r2*z differs on about one output coordinate in six.
// Device: __dmul_rn / __dadd_rn / __dsub_rn (arith.h's mul_ / add_ / sub_) and __ddiv_rn / __dsqrt_rn; host: plain
// operators under -ffp-contract=off.
//
// sin and cos are glibc's, which the device cannot reproduce (DESIGN §4.4); but their argument takes only a handful
// of values.  With u = 2^-53 (unit roundoff) and t = fl(theta) (|t| normal): n carries a relative error of at most
// 2u (the sum of squares of non-negative terms ~2u, halved by the square root, plus u for its rounding), c_i / n and
// t * (.) add u each, and a adds 2u like n.  So |a - |t|| <= 6u |t| (1 + O(u)) < 6 ulp(|t|) -- or 12 steps of the
// double grid when a crosses the binade boundary below |t|, where the ulp halves.  The host therefore evaluates
// sin(v/2)/v and cos(v/2) with its own libm for every double v within kVcorrHalf = 16 grid steps of |t| (margin
// > 2.5x over the bound; 2 x 33 doubles per angle), and the device looks them up by the bit distance of a from |t|.
// The bound assumes the squares do not under- or overflow.  For float32 input they never do (|c| <= 3.4e38, squares
// >= 2e-90); for float64 input an overflowing n (|x| or |y| above ~1e154) gives a = 0, whose cos is exactly 1 and is
// handled below, and an underflowing one (|x|, |y| below ~1e-154, not both zero) can give a finite angle outside the
// table: the device raises an error flag, and the call fails with MADICP_ERR_STATE -- it never produces a different
// point.  NaN and infinite angles (x = y = 0 gives n = 0 and c / n = NaN) give NaN rows, as scipy's sin(NaN)/NaN does.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "arith.h"

namespace madicp {

constexpr int kVcorrHalf = 16;  // table entries on each side of |fl(theta)|

struct VcorrTable {
  double theta;                   // the angle, fl(theta)
  double center;                  // |theta|: where the rotation angles a of the points lie
  double s[2 * kVcorrHalf + 1];   // sin(v/2)/v at the double k steps from center, k = -16..16 (NaN where v is not >= 0)
  double w[2 * kVcorrHalf + 1];   // cos(v/2)
};

// division, square root and bit pattern next to arith.h's mul_ / add_ / sub_
#if defined(__CUDA_ARCH__)
MADICP_HD double vc_div(double a, double b) { return __ddiv_rn(a, b); }
MADICP_HD double vc_sqrt(double a) { return __dsqrt_rn(a); }
MADICP_HD int64_t vc_bits(double a) { return __double_as_longlong(a); }
#else
MADICP_HD double vc_div(double a, double b) { return a / b; }
MADICP_HD double vc_sqrt(double a) { return sqrt(a); }
MADICP_HD int64_t vc_bits(double a) {
  int64_t b;
  memcpy(&b, &a, sizeof(b));
  return b;
}
#endif

// The table of one angle, with the host's libm (host code only).
inline void vcorr_table_fill(double theta, VcorrTable* t) {
  t->theta = theta;
  t->center = fabs(theta);
  const int64_t c = vc_bits(t->center);
  for (int k = -kVcorrHalf; k <= kVcorrHalf; ++k) {
    const int64_t b = c + k;
    double v = NAN;
    if (b >= 0) memcpy(&v, &b, sizeof(v));
    t->s[k + kVcorrHalf] = sin(v / 2) / v;
    t->w[k + kVcorrHalf] = cos(v / 2);
  }
}

// The corrected point of (x, y, z) (the field values as float64).  Returns false, and leaves the point alone, when its
// rotation angle is finite and outside the table (see above).
MADICP_HD bool vcorr_apply(const VcorrTable& t, double& x, double& y, double& z) {
  const double c0 = sub_(mul_(y, 1.0), mul_(z, 0.0));
  const double c1 = sub_(mul_(z, 0.0), mul_(x, 1.0));
  const double c2 = sub_(mul_(x, 0.0), mul_(y, 0.0));
  const double n = vc_sqrt(add_(add_(mul_(c0, c0), mul_(c1, c1)), mul_(c2, c2)));
  const double r0 = mul_(t.theta, vc_div(c0, n)), r1 = mul_(t.theta, vc_div(c1, n)), r2 = mul_(t.theta, vc_div(c2, n));
  const double a = vc_sqrt(add_(add_(mul_(r0, r0), mul_(r1, r1)), mul_(r2, r2)));
  const double a2 = mul_(a, a);
  double s, w;
  if (!(a < INFINITY)) {  // NaN or inf: sin(a/2)/a and cos(a/2) are NaN
    s = w = NAN;
  } else if (a == 0.0) {
    s = 0.5;
    w = 1.0;
  } else {
    const int64_t k = vc_bits(a) - vc_bits(t.center);
    if (k < -kVcorrHalf || k > kVcorrHalf) return false;
    s = a <= 1e-3 ? add_(sub_(0.5, vc_div(a2, 48.0)), vc_div(mul_(a2, a2), 3840.0)) : t.s[k + kVcorrHalf];
    w = t.w[k + kVcorrHalf];
  }
  const double qx = mul_(s, r0), qy = mul_(s, r1), qz = mul_(s, r2), qw = w;
  const double x2 = mul_(qx, qx), y2 = mul_(qy, qy), z2 = mul_(qz, qz), w2 = mul_(qw, qw);
  const double xy = mul_(qx, qy), xz = mul_(qx, qz), xw = mul_(qx, qw);
  const double yz = mul_(qy, qz), yw = mul_(qy, qw), zw = mul_(qz, qw);
  const double m00 = add_(sub_(sub_(x2, y2), z2), w2);
  const double m01 = mul_(2.0, sub_(xy, zw));
  const double m02 = mul_(2.0, add_(xz, yw));
  const double m10 = mul_(2.0, add_(xy, zw));
  const double m11 = add_(sub_(add_(-x2, y2), z2), w2);
  const double m12 = mul_(2.0, sub_(yz, xw));
  const double m20 = mul_(2.0, sub_(xz, yw));
  const double m21 = mul_(2.0, add_(yz, xw));
  const double m22 = add_(add_(sub_(-x2, y2), z2), w2);
  const double ox = add_(add_(add_(0.0, mul_(m00, x)), mul_(m02, z)), mul_(m01, y));
  const double oy = add_(add_(add_(0.0, mul_(m10, x)), mul_(m12, z)), mul_(m11, y));
  const double oz = add_(add_(add_(0.0, mul_(m20, x)), mul_(m22, z)), mul_(m21, y));
  x = ox;
  y = oy;
  z = oz;
  return true;
}

}  // namespace madicp
