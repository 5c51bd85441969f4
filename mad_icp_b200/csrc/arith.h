// arith.h -- single-source FP64 primitives shared by host C++ and sm_90a device code.
//
// Bit-exact correspondence indices require the descent predicate
//   ((q - mean) . dir) < 0                        (reference: tools/mad_tree.cpp:148)
// to round identically on the host (flat-tree builder, facade) and on the GPU.  Every
// function here therefore has ONE fixed operand order and never forms an FMA:
//   * device code is compiled with -fmad=false and additionally spells the predicate
//     chain with __dmul_rn/__dadd_rn/__dsub_rn (which ptxas never contracts);
//   * host code is compiled with -ffp-contract=off and without -march=native.
// The 3-term sum order is ((a0*b0 + a1*b1) + a2*b2) everywhere (DESIGN.md "arithmetic").
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define MADICP_HD __host__ __device__ __forceinline__
#else
#define MADICP_HD inline
#endif

namespace madicp {

#if defined(__CUDA_ARCH__)
MADICP_HD double mul_(double a, double b) { return __dmul_rn(a, b); }
MADICP_HD double add_(double a, double b) { return __dadd_rn(a, b); }
MADICP_HD double sub_(double a, double b) { return __dsub_rn(a, b); }
#else
MADICP_HD double mul_(double a, double b) { return a * b; }
MADICP_HD double add_(double a, double b) { return a + b; }
MADICP_HD double sub_(double a, double b) { return a - b; }
#endif

// (a0*b0 + a1*b1) + a2*b2
MADICP_HD double dot3(double a0, double a1, double a2, double b0, double b1, double b2) {
  return add_(add_(mul_(a0, b0), mul_(a1, b1)), mul_(a2, b2));
}
// split-plane side value of query q against (mean, dir):  (q - mean) . dir
MADICP_HD double plane_side(double qx, double qy, double qz, double mx, double my, double mz, double dx, double dy,
                            double dz) {
  return dot3(sub_(qx, mx), sub_(qy, my), sub_(qz, mz), dx, dy, dz);
}
MADICP_HD double norm3(double x, double y, double z) { return sqrt(dot3(x, y, z, x, y, z)); }

// Pose stored row-major 3x4: X[r*4+c], c<3 rotation, c==3 translation.
// y = R*p + t with each row as a dot3, translation added last (reference: odometry/mad_icp.cpp:78).
MADICP_HD void iso_apply(const double* X, double px, double py, double pz, double& ox, double& oy, double& oz) {
  ox = add_(dot3(X[0], X[1], X[2], px, py, pz), X[3]);
  oy = add_(dot3(X[4], X[5], X[6], px, py, pz), X[7]);
  oz = add_(dot3(X[8], X[9], X[10], px, py, pz), X[11]);
}

// C = A*B for poses (row-major 3x4): R = Ra*Rb, t = Ra*tb + ta  (reference: odometry/mad_icp.cpp:116)
MADICP_HD void iso_mul(const double* A, const double* B, double* C) {
#pragma unroll
  for (int r = 0; r < 3; ++r) {
#pragma unroll
    for (int c = 0; c < 3; ++c) C[r * 4 + c] = dot3(A[r * 4], A[r * 4 + 1], A[r * 4 + 2], B[c], B[4 + c], B[8 + c]);
    C[r * 4 + 3] = add_(dot3(A[r * 4], A[r * 4 + 1], A[r * 4 + 2], B[3], B[7], B[11]), A[r * 4 + 3]);
  }
}

}  // namespace madicp
