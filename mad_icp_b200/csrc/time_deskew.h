// time_deskew.h -- the chunk of a point from its own time stamp (madicp_times_t, include/madicp_b200.h), ONE rule for
// host C++ and sm_90a device code:
//   u = (tau - t_end) * scale;  s = rint(((-u) * sensor_hz) * (CHUNKS - 1));  k = CHUNKS - 1 - clamp(s, 0, CHUNKS - 1)
// in float64, no FMA (mul_ / sub_ of arith.h), rint rounding half to even on both sides.  NaN clamps to 0 (k = CHUNKS - 1)
// so that a chunk is always a valid table index; a kept NaN or infinite stamp fails the call before its point is used.
// The default t_end is the largest kept stamp: a max is exact and order-free, so the device reduces it through an
// integer-ordered key (time_key) with atomics in any order and gets the host's value.
#pragma once
#include <math.h>
#include <stdint.h>
#include <string.h>

#include "arith.h"

namespace madicp {

constexpr int kTimeChunks = 1024;  // tools/constants.h:31
constexpr int kTimeNone = 0, kTimeU32 = 1, kTimeF32 = 2, kTimeF64 = 3;  // MADICP_TIME_*

MADICP_HD int time_size(int type) { return type == kTimeF64 ? 8 : 4; }

MADICP_HD int time_chunk(double tau, double t_end, double scale, double sensor_hz) {
  const double u = mul_(sub_(tau, t_end), scale);
  const double s = rint(mul_(mul_(-u, sensor_hz), double(kTimeChunks - 1)));
  const double c = s > 0.0 ? (s < double(kTimeChunks - 1) ? s : double(kTimeChunks - 1)) : 0.0;
  return kTimeChunks - 1 - int(c);
}

// a < b  <=>  time_key(a) < time_key(b) for finite doubles (-0.0 below +0.0); never 0 for a finite value
MADICP_HD unsigned long long time_key(double t) {
#if defined(__CUDA_ARCH__)
  const unsigned long long b = (unsigned long long) __double_as_longlong(t);
#else
  unsigned long long b;
  memcpy(&b, &t, sizeof(b));
#endif
  return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
MADICP_HD double time_of_key(unsigned long long k) {
  const unsigned long long b = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
#if defined(__CUDA_ARCH__)
  return __longlong_as_double((long long) b);
#else
  double t;
  memcpy(&t, &b, sizeof(t));
  return t;
#endif
}

}  // namespace madicp
