// records.hpp -- host side of madicp_points_t (include/madicp_b200.h): validation, field reads, the range gate
// (range_gate.h) with its bounds rounded to the field type, and the optional vertical-angle correction
// (madicp_vcorr_t, vertical_correction.h).  Shared by gpu_tree.cu, ingest.cpp and the facade.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <cstring>
#include <string>

#include "../../include/madicp_b200.h"
#include "range_gate.h"
#include "time_deskew.h"
#include "vertical_correction.h"

namespace madicp {
void set_error(const std::string& msg);

// the packed N x 3 cloud of madicp_ingest / madicp_stage_cloud / madtree_gpu_build_batch
inline madicp_points_t packed_points(const void* xyz, int64_t n, int is_f32) {
  madicp_points_t d{};
  const int32_t e = is_f32 ? 4 : 8;
  d.data = xyz;
  d.n = n;
  d.stride = 3 * e;
  d.offset[0] = 0; d.offset[1] = e; d.offset[2] = 2 * e;
  d.is_f32 = is_f32 ? 1 : 0;
  d.range_mode = kGateNone;
  return d;
}
inline bool points_gated(const madicp_points_t& d) { return d.range_mode != kGateNone || d.drop_nan; }
// bytes from the first record's start to the end of the last record's last field: what is read (and uploaded), so
// that a view whose last record is cut short (e.g. the x/y/z columns of a larger array) is never read past its end
inline size_t points_bytes(const madicp_points_t& d) {
  const int64_t e = d.is_f32 ? 4 : 8;
  const int64_t end = std::max(d.offset[0], std::max(d.offset[1], d.offset[2])) + e;
  return size_t((d.n - 1) * d.stride + end);
}
// the correction of a nullable madicp_vcorr_t: disabled, or enabled with its angle (the reserved field ignored)
inline madicp_vcorr_t vcorr_of(const madicp_vcorr_t* v) {
  madicp_vcorr_t o{};
  if (v && v->enabled) {
    o.angle = v->angle;
    o.enabled = 1;
  }
  return o;
}
// the same scan as far as the device is concerned: equal descriptors and equal corrections (angles equal bit for bit)
inline bool same_points(const madicp_points_t& a, const madicp_vcorr_t& va, const madicp_points_t& b,
                        const madicp_vcorr_t& vb) {
  if (va.enabled != vb.enabled || (va.enabled && std::memcmp(&va.angle, &vb.angle, sizeof(double)) != 0)) return false;
  return a.data == b.data && a.n == b.n && a.stride == b.stride && a.offset[0] == b.offset[0] && a.offset[1] == b.offset[1] &&
         a.offset[2] == b.offset[2] && (a.is_f32 != 0) == (b.is_f32 != 0) && a.min_range == b.min_range &&
         a.max_range == b.max_range && a.range_mode == b.range_mode && (a.drop_nan != 0) == (b.drop_nan != 0);
}

// MADICP_OK, or MADICP_ERR_INVALID with a message naming `fn`
inline int check_points(const madicp_points_t* d, const char* fn) {
  auto bad = [fn](const std::string& why) {
    set_error(std::string(fn) + ": " + why);
    return MADICP_ERR_INVALID;
  };
  if (!d) return bad("null descriptor");
  if (!d->data) return bad("null data");
  if (d->n < 1 || d->n > (int64_t(1) << 24)) return bad("n must be 1..2^24 records");
  const int64_t e = d->is_f32 ? 4 : 8;
  if (d->stride < 1 || d->stride > 65536 || d->stride % e)
    return bad("stride must be a positive multiple of the field size, at most 65536 bytes");
  for (int c = 0; c < 3; ++c) {
    if (d->offset[c] < 0 || d->offset[c] + e > d->stride) return bad("field " + std::to_string(c) + " does not fit the stride");
    if (d->offset[c] % e) return bad("field " + std::to_string(c) + " offset is not a multiple of the field size");
  }
  if (std::isnan(d->min_range) || std::isnan(d->max_range)) return bad("NaN range bound");
  if (d->min_range > d->max_range) return bad("min_range > max_range");
  if (d->range_mode < kGateNone || d->range_mode > kGateStrict) return bad("range_mode must be 0, 1 or 2");
  return MADICP_OK;
}
// MADICP_OK, or MADICP_ERR_INVALID with a message naming `fn`: an enabled correction needs a finite angle
inline int check_vcorr(const madicp_vcorr_t* v, const char* fn) {
  if (v && v->enabled && !std::isfinite(v->angle)) {
    set_error(std::string(fn) + ": the vertical correction angle must be finite");
    return MADICP_ERR_INVALID;
  }
  return MADICP_OK;
}

// The time field of a nullable madicp_times_t (time_deskew.h): none, or its layout and constants (reserved ignored)
inline madicp_times_t times_of(const madicp_times_t* t) {
  madicp_times_t o{};
  if (t && t->type != kTimeNone) {
    o = *t;
    o.reserved = 0;
    if (!o.has_t_end) o.t_end = 0.0;
    o.has_t_end = o.has_t_end ? 1 : 0;
  }
  return o;
}
// MADICP_OK, or MADICP_ERR_INVALID with a message naming `fn`: a time field must fit the stride, be aligned for its
// type, and come with a finite scale > 0 and a finite t_end (when given)
inline int check_times(const madicp_times_t* t, const madicp_points_t* d, const char* fn) {
  if (!t || t->type == kTimeNone) return MADICP_OK;
  auto bad = [fn](const std::string& why) {
    set_error(std::string(fn) + ": " + why);
    return MADICP_ERR_INVALID;
  };
  if (t->type < kTimeU32 || t->type > kTimeF64) return bad("time field type must be 0 (none), 1 (uint32), 2 (float32) or 3 (float64)");
  const int64_t e = time_size(t->type);
  if (t->offset < 0 || t->offset + e > d->stride) return bad("time field does not fit the stride");
  if (t->offset % e || d->stride % e) return bad("time field is misaligned for its type (offset and stride must be multiples of its size)");
  if (!(t->scale > 0.0) || !std::isfinite(t->scale)) return bad("time scale must be finite and > 0");
  if (t->has_t_end && !std::isfinite(t->t_end)) return bad("time t_end must be finite");
  return MADICP_OK;
}
// points_bytes with the time field: what a scan with one is read up to
inline size_t points_bytes(const madicp_points_t& d, const madicp_times_t& t) {
  if (t.type == kTimeNone) return points_bytes(d);
  const size_t end = size_t((d.n - 1) * d.stride + t.offset + time_size(t.type));
  return std::max(points_bytes(d), end);
}
// record i's time as float64 (exact for every type)
inline double time_at(const madicp_points_t& d, const madicp_times_t& t, int64_t i) {
  const char* r = static_cast<const char*>(d.data) + i * d.stride + t.offset;
  if (t.type == kTimeF64) {
    double v;
    std::memcpy(&v, r, 8);
    return v;
  }
  if (t.type == kTimeF32) {
    float v;
    std::memcpy(&v, r, 4);
    return double(v);
  }
  uint32_t v;
  std::memcpy(&v, r, 4);
  return double(v);
}

// The gate of one descriptor in field type T, and the correction (nullable table) of its kept points
template <class T>
struct RecReader {
  const char* base;
  int64_t stride;
  int32_t off[3];
  T lo, hi;
  int mode, drop_nan;
  bool gated;
  const VcorrTable* vc;
  explicit RecReader(const madicp_points_t& d, const VcorrTable* vc_table = nullptr)
      : base(static_cast<const char*>(d.data)), stride(d.stride), off{d.offset[0], d.offset[1], d.offset[2]},
        lo(T(d.min_range)), hi(T(d.max_range)), mode(d.range_mode), drop_nan(d.drop_nan), gated(points_gated(d)),
        vc(vc_table) {}
  void xyz(int64_t i, T& x, T& y, T& z) const {
    const char* r = base + i * stride;
    std::memcpy(&x, r + off[0], sizeof(T));
    std::memcpy(&y, r + off[1], sizeof(T));
    std::memcpy(&z, r + off[2], sizeof(T));
  }
  bool keep(T x, T y, T z) const { return !gated || range_keep<T>(x, y, z, lo, hi, mode, drop_nan); }
  // Record i: whether the gate keeps it and, when it does, its point as float64, corrected.  `bad` is set when the
  // correction's angle falls outside the table (the point is then not the reader's: the caller fails).
  bool kept_point(int64_t i, double& x, double& y, double& z, bool& bad) const {
    T fx, fy, fz;
    xyz(i, fx, fy, fz);
    if (!keep(fx, fy, fz)) return false;
    x = double(fx); y = double(fy); z = double(fz);
    if (vc && !vcorr_apply(*vc, x, y, z)) bad = true;
    return true;
  }
};

}  // namespace madicp
