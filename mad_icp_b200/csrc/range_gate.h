// range_gate.h -- the dataset readers' point filter as ONE predicate shared by host C++ and sm_90a device code.
//
// The readers drop points before the scan reaches Pipeline::compute:
//   KITTI      apps/utils/kitti_reader.py:82-88     norms = np.linalg.norm(cloud[:, :3], axis=1)
//                                                  keep  = (norms >= min_range) & (norms <= max_range)
//   PointCloud2 apps/utils/point_cloud2.py:77-87    drop rows with a NaN coordinate, then
//                                                  keep  = (norms > min_range) & (norms < max_range)
// np.linalg.norm over the rows of a float32 N x 3 array is sqrt((x*x + y*y) + z*z) with every operation rounded in
// float32 (float64 input: the same order in double), and a Python float bound is compared in the array's type.  So
// the norm is spelled here with that order and without FMA (__fmul_rn / __fadd_rn / __fsqrt_rn on the device, plain
// operators under -ffp-contract=off on the host), and the bounds arrive already rounded to the field type.
#pragma once
#include <math.h>

#include "arith.h"

namespace madicp {

// range_mode of madicp_points_t
constexpr int kGateNone = 0, kGateInclusive = 1, kGateStrict = 2;

#if defined(__CUDA_ARCH__)
MADICP_HD float gate_mul(float a, float b) { return __fmul_rn(a, b); }
MADICP_HD float gate_add(float a, float b) { return __fadd_rn(a, b); }
MADICP_HD float gate_sqrt(float a) { return __fsqrt_rn(a); }
MADICP_HD double gate_mul(double a, double b) { return __dmul_rn(a, b); }
MADICP_HD double gate_add(double a, double b) { return __dadd_rn(a, b); }
MADICP_HD double gate_sqrt(double a) { return __dsqrt_rn(a); }
#else
MADICP_HD float gate_mul(float a, float b) { return a * b; }
MADICP_HD float gate_add(float a, float b) { return a + b; }
MADICP_HD float gate_sqrt(float a) { return sqrtf(a); }
MADICP_HD double gate_mul(double a, double b) { return a * b; }
MADICP_HD double gate_add(double a, double b) { return a + b; }
MADICP_HD double gate_sqrt(double a) { return sqrt(a); }
#endif

// Does the point survive the reader's filter?  lo / hi: the bounds rounded to T once.  A NaN norm fails every
// comparison, so with a gate on a NaN coordinate drops the point whether or not drop_nan is set.
template <class T>
MADICP_HD bool range_keep(T x, T y, T z, T lo, T hi, int mode, int drop_nan) {
  if (drop_nan && (x != x || y != y || z != z)) return false;
  if (mode == kGateNone) return true;
  const T r = gate_sqrt(gate_add(gate_add(gate_mul(x, x), gate_mul(y, y)), gate_mul(z, z)));
  return mode == kGateInclusive ? (lo <= r && r <= hi) : (lo < r && r < hi);
}

}  // namespace madicp
