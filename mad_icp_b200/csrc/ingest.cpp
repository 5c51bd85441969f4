// ingest.cpp -- host-side preparation of an incoming scan before its tree is built (SURVEY 8f, next-3).
//
// madicp_deskew is the reference's Pipeline::deskew (odometry/pipeline.cpp:79-123): the points are sorted
// by azimuth, the sweep is cut into 1024 chunks, every chunk gets the pose interpolated from the last
// relative motion, and the cloud is rewritten IN SORTED ORDER with those poses applied.  The order matters
// downstream (the tree's sums run in array order), so the result must be the reference's permutation
// exactly -- and equal azimuths are the rule in lidar data (the beams of one firing column), so the
// order std::sort happens to leave among them is part of the result.  That order depends only on the
// sequence of comparison outcomes, not on what is being moved: the same std::sort over 16-byte
// (azimuth, index) records takes the same decisions as the reference's over its 32-byte (azimuth, point)
// pairs and ends with the same permutation, at half the traffic.  Everything else (atan2 per point, the
// chunk poses, the transform) is a pure per-point function and is spread over the worker pool.  The
// reference spends ~10 ms per 131k-point scan here on one core.
#include <algorithm>
#include <chrono>
#include <cmath>
#include <functional>
#include <memory>
#include <cstdio>
#include <cstdlib>
#include <cstdint>
#include <cstring>
#include <string>
#include <utility>
#include <vector>

#include "../../include/madicp_b200_debug.h"
#include "host_pool.hpp"
#include "pose_math.h"
#include "records.hpp"

namespace {
using madicp_host::default_init_allocator;
using madicp_host::for_chunks;
using madicp_pose::Pose;

constexpr int kChunks = 1024;  // tools/constants.h:31

struct Item {
  double key;
  int32_t idx;
  int32_t pad;
};
struct P3 {
  double v[3];
};

template <class T>
using RawVec = std::vector<T, default_init_allocator<T>>;

// ---------------------------------------------------------------------------------------------
// std::sort's outcome, in parallel.  GNU libstdc++ sorts with introsort: quicksort steps (pivot = median
// of the second, middle and last element, moved to the front; Hoare-style unguarded partition) down to
// ranges of 16, heapsort when a range has used up 2*floor(log2 n) levels, then one insertion-sort pass
// over everything.  What it leaves among equal keys is decided by those steps, so they are restated here
// step for step -- but the two sides of a partition never interact again, so they go to different
// threads, and the closing insertion sort, being stable, gives the same array whether it runs over
// everything or over each partition-ordered range separately.  tests/test_pybind_api.py checks the
// permutation against std::sort itself (madicp_debug_sort_check) on keys with many ties.
struct KeyLess {
  bool operator()(const Item& x, const Item& y) const { return x.key < y.key; }
};
inline void median_to_first(Item* result, Item* a, Item* b, Item* c) {
  KeyLess lt;
  if (lt(*a, *b)) {
    if (lt(*b, *c)) std::swap(*result, *b);
    else if (lt(*a, *c)) std::swap(*result, *c);
    else std::swap(*result, *a);
  } else if (lt(*a, *c)) std::swap(*result, *a);
  else if (lt(*b, *c)) std::swap(*result, *c);
  else std::swap(*result, *b);
}
inline Item* partition_step(Item* first, Item* last) {
  KeyLess lt;
  Item* mid = first + (last - first) / 2;
  median_to_first(first, first + 1, mid, last - 1);
  Item* lo = first + 1;
  Item* hi = last;
  for (;;) {
    while (lt(*lo, *first)) ++lo;
    --hi;
    while (lt(*first, *hi)) --hi;
    if (!(lo < hi)) return lo;
    std::swap(*lo, *hi);
    ++lo;
  }
}
void quick_phase(Item* first, Item* last, int depth_limit) {  // the loop that precedes the insertion pass
  while (last - first > 16) {
    if (depth_limit == 0) {
      std::partial_sort(first, last, last, KeyLess());  // make_heap + sort_heap over the range
      return;
    }
    --depth_limit;
    Item* cut = partition_step(first, last);
    quick_phase(cut, last, depth_limit);
    last = cut;
  }
}
void insertion_pass(Item* first, Item* last) {  // stable
  KeyLess lt;
  for (Item* i = first + (first != last); i < last; ++i) {
    const Item v = *i;
    Item* j = i;
    while (j > first && lt(v, *(j - 1))) {
      *j = *(j - 1);
      --j;
    }
    *j = v;
  }
}
struct Range {
  Item *first, *last;
  int depth_limit;
  bool done;  // heap-sorted or at most 16 long: only the insertion pass is left
};
void sort_like_std(Item* first, Item* last, int threads) {
  const ptrdiff_t n = last - first;
  if (n < 2) return;
  int lg = 0;
  for (ptrdiff_t m = n; m > 1; m >>= 1) ++lg;
  std::vector<Range> ranges{Range{first, last, 2 * lg, false}};
  // The first splits are done here, one after the other (a pass over the data each), until there are
  // about two ranges per thread; everything below them is then finished in ONE parallel section.  (Handing
  // the early rounds to the pool as well would save a fraction of a millisecond on an idle machine and
  // cost several wake-ups of every worker on a busy or virtualised one.)
  const ptrdiff_t cutoff = std::max<ptrdiff_t>(4096, n / (2 * std::max(threads, 1)));
  for (size_t r = 0; r < ranges.size(); ++r) {
    while (!ranges[r].done && ranges[r].last - ranges[r].first > cutoff) {
      Range& R = ranges[r];
      if (R.depth_limit == 0) {
        std::partial_sort(R.first, R.last, R.last, KeyLess());
        R.done = true;
        break;
      }
      --R.depth_limit;
      Item* cut = partition_step(R.first, R.last);
      const Range right{cut, R.last, R.depth_limit, false};
      R.last = cut;
      ranges.push_back(right);  // (invalidates R: it is re-read at the top of the loop)
    }
  }
  for_chunks(threads, ranges.size(), 1, [&](size_t r0, size_t) {
    Range& R = ranges[r0];
    if (!R.done) quick_phase(R.first, R.last, R.depth_limit);
    insertion_pass(R.first, R.last);
  });
}

// sorted keys -> chunk number of every position (the reference advances by at most one chunk per point)
void sweep(const Item* it, int64_t n, double resolution, RawVec<int32_t>& cid, int32_t& last) {
  double angle = M_PI - resolution;
  int32_t c = 0;
  for (int64_t i = n - 1; i >= 0; --i) {
    if (it[i].key < angle) {
      angle -= resolution;
      ++c;
    }
    cid[size_t(i)] = c;
  }
  last = c;
}

// The pose half of the deskew: the relative motion of the last two poses as a constant twist (pipeline.cpp:80-86), and
// the pose of every chunk c < count, handed to out(c, pose) in chunk order (t accumulates as in the reference).
template <class F>
void chunk_poses(const double T_prev[12], const double T_now[12], double sensor_hz, int count, F&& out) {
  const double ts = 1. / sensor_hz;
  Pose a, b;
  std::memcpy(a.m, T_prev, sizeof(a.m));
  std::memcpy(b.m, T_now, sizeof(b.m));
  const Pose rel = madicp_pose::poseMul(madicp_pose::poseInverse(a), b);
  double w[3];
  madicp_pose::logSO3(rel, w);
  const double vel[6] = {rel.m[3] / ts, rel.m[7] / ts, rel.m[11] / ts, w[0] / ts, w[1] / ts, w[2] / ts};
  const double delta = ts / double(kChunks - 1);
  double t = -ts;
  for (int c = 0; c < count; ++c) {
    const double tr[3] = {vel[0] * t, vel[1] * t, vel[2] * t}, ro[3] = {vel[3] * t, vel[4] * t, vel[5] * t};
    out(c, madicp_pose::poseFromTwist(tr, ro));
    t += delta;
  }
}

}  // namespace

extern "C" int madicp_deskew(double* points_xyz, int64_t n, const double T_prev[12], const double T_now[12], double sensor_hz,
                             int num_threads) {
  if (!points_xyz || !T_prev || !T_now || n <= 0 || n > (int64_t(1) << 30) || !(sensor_hz > 0.0)) {
    madicp::set_error("madicp_deskew: bad arguments");
    return MADICP_ERR_INVALID;
  }
  int threads = num_threads < 1 ? 1 : (num_threads > 64 ? 64 : num_threads);
  if (n < 20000) threads = 1;
  const size_t un = size_t(n);
  const double resolution = 2 * M_PI / double(kChunks);

  madicp_host::HotScope hot;  // the serial first splits of the sort sit between two parallel sections
  const bool timing = std::getenv("MADTREE_TIMING") != nullptr;
  auto now = []() { return std::chrono::steady_clock::now(); };
  auto ms = [](std::chrono::steady_clock::time_point x, std::chrono::steady_clock::time_point y) {
    return std::chrono::duration<double, std::milli>(y - x).count();
  };
  const auto t0 = now();
  // azimuth of every point (pipeline.cpp:91-95)
  // (the same pass keeps a copy of the points: the result is written over the input in another order)
  RawVec<Item> items(un);
  RawVec<P3> in(un);
  for_chunks(threads, un, 8192, [&](size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) {
      items[i] = Item{std::atan2(points_xyz[3 * i + 1], points_xyz[3 * i]), int32_t(i), 0};
      std::memcpy(in[i].v, points_xyz + 3 * i, sizeof(double) * 3);
    }
  });
  const auto t1 = now();

  // the reference's sort (pipeline.cpp:97-99), on records that carry an index instead of the point
  if (threads > 1) sort_like_std(items.data(), items.data() + un, threads);
  else std::sort(items.begin(), items.end(), KeyLess());

  const auto t2 = now();
  // which chunk each sorted position falls in, then the chunk poses (t accumulates as in the reference)
  RawVec<int32_t> cid(un);
  int32_t last = 0;
  sweep(items.data(), n, resolution, cid, last);
  std::vector<Pose> meas(size_t(last) + 1);
  chunk_poses(T_prev, T_now, sensor_hz, last + 1, [&](int c, const Pose& m) { meas[size_t(c)] = m; });
  // (*curr_cloud)[i] = meas_pose_to_robot * sorted[i].second  (pipeline.cpp:121)
  for_chunks(threads, un, 8192, [&](size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) madicp_pose::poseApply(meas[size_t(cid[i])], in[size_t(items[i].idx)].v, points_xyz + 3 * i);
  });
  if (timing)
    std::fprintf(stderr, "madicp_deskew: n=%lld threads=%d azimuths %.2f ms, sort %.2f ms%s, sweep+poses+apply %.2f ms\n", (long long) n,
                 threads, ms(t0, t1), ms(t1, t2), "", ms(t2, now()));
  return MADICP_OK;
}

// The host half of the device-side ingest (gpu_tree.cu, madicp_ingest): everything of Pipeline::deskew that decides
// an ORDER or calls libm -- azimuths (atan2), the reference's sort permutation, the chunk of every sorted position,
// the chunk poses (sin/cos inside the exponential map) -- and nothing that touches the points' values: the gather,
// the float -> double conversion and the rigid transform run on the device.  It comes in two halves.
//
// The order half (madicp_deskew_order) depends on the points alone: the azimuths, their sort (ties included) and each
// sorted position's chunk -- the sweep compares the azimuths with an angle that drops by `resolution` per chunk whatever
// the motion.  So it can run for a scan long before the poses it will be deskewed with exist (madicp_plan_points).
// The records are read through their descriptor and the range gate (records.hpp) is applied in the azimuth pass: the
// sort sees the kept points in record order, exactly the cloud the reader would have handed over.  With a vertical
// correction (vc != nullptr, vertical_correction.h) the azimuths are those of the corrected points, as the reader
// corrects before the pipeline deskews; MADICP_ERR_STATE (no message) when a rotation angle falls outside the table.
// perm[i] = record index of the kept point at sorted position i; chunk[i] = its pose; *n_chunks = number of chunk
// poses the pose half must produce (0 when nothing is kept); *n_kept = number of kept points (entries of perm / chunk).
// num_threads == 1 runs on the calling thread alone, without touching the shared pool (several scans' order halves
// run side by side on threads of their own, and a tree build's libm sections need the pool meanwhile).
int madicp_deskew_order(const madicp_points_t& pts, const madicp::VcorrTable* vc, int num_threads, int32_t* perm,
                        uint16_t* chunk, int* n_chunks, int64_t* n_kept) {
  const int64_t n_rec = pts.n;
  if (!pts.data || n_rec <= 0 || n_rec > (int64_t(1) << 30)) {
    madicp::set_error("madicp_ingest: bad arguments");
    return MADICP_ERR_INVALID;
  }
  int threads = num_threads < 1 ? 1 : (num_threads > 64 ? 64 : num_threads);
  if (n_rec < 20000) threads = 1;
  auto each = [threads](size_t n, size_t grain, auto&& fn) {  // fn(c0, c1) over [0, n): the pool only when threaded
    if (threads > 1) for_chunks(threads, n, grain, fn);
    else fn(size_t(0), n);
  };
  const double resolution = 2 * M_PI / double(kChunks);
  std::unique_ptr<madicp_host::HotScope> hot(threads > 1 ? new madicp_host::HotScope : nullptr);
  RawVec<Item> items(static_cast<size_t>(n_rec));
  auto azimuths = [&](auto zero) {  // (pad = 1: the record survives the gate; 2: ... but its correction failed)
    using T = decltype(zero);
    const madicp::RecReader<T> rd(pts, vc);
    each(size_t(n_rec), 8192, [&](size_t c0, size_t c1) {
      for (size_t i = c0; i < c1; ++i) {
        double x = 0, y = 0, z = 0;
        bool bad = false;
        const bool kept = rd.kept_point(int64_t(i), x, y, z, bad);
        items[i] = Item{std::atan2(y, x), int32_t(i), bad ? 2 : (kept ? 1 : 0)};
      }
    });
  };
  if (pts.is_f32) azimuths(0.0f);
  else azimuths(0.0);
  size_t un = size_t(n_rec);
  if (madicp::points_gated(pts) || vc) {  // the kept records, in record order
    un = 0;
    for (size_t i = 0; i < size_t(n_rec); ++i) {
      if (items[i].pad == 2) return MADICP_ERR_STATE;
      if (items[i].pad) items[un++] = items[i];
    }
  }
  *n_kept = int64_t(un);
  *n_chunks = 0;
  if (un == 0) return MADICP_OK;
  const int64_t n = int64_t(un);
  if (threads > 1) sort_like_std(items.data(), items.data() + un, threads);
  else std::sort(items.begin(), items.begin() + ptrdiff_t(un), KeyLess());
  RawVec<int32_t> cid(un);
  int32_t last = 0;
  sweep(items.data(), n, resolution, cid, last);
  if (last >= 65535) {
    madicp::set_error("madicp_ingest: more than 65535 deskew chunks");
    return MADICP_ERR_INVALID;
  }
  each(un, 16384, [&](size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) {
      perm[i] = items[i].idx;
      chunk[i] = uint16_t(cid[i]);
    }
  });
  *n_chunks = last + 1;
  return MADICP_OK;
}

// The pose half: the n_chunks chunk poses (n_chunks x 12 row-major) of the motion from T_prev to T_now.
void madicp_deskew_poses(const double T_prev[12], const double T_now[12], double sensor_hz, int n_chunks, double* poses) {
  chunk_poses(T_prev, T_now, sensor_hz, n_chunks,
              [poses](int c, const Pose& m) { std::memcpy(poses + size_t(c) * 12, m.m, sizeof(double) * 12); });
}

// Both halves in a row: perm / chunk / *n_kept as madicp_deskew_order, poses: (*n_poses) x 12 row-major.
int madicp_deskew_plan(const madicp_points_t& pts, const madicp::VcorrTable* vc, const double T_prev[12],
                       const double T_now[12], double sensor_hz, int num_threads, int32_t* perm, uint16_t* chunk,
                       double* poses, int* n_poses, int64_t* n_kept) {
  if (!pts.data || !T_prev || !T_now || pts.n <= 0 || pts.n > (int64_t(1) << 30) || !(sensor_hz > 0.0)) {
    madicp::set_error("madicp_ingest: bad arguments");
    return MADICP_ERR_INVALID;
  }
  *n_poses = 0;
  const int rc = madicp_deskew_order(pts, vc, num_threads, perm, chunk, n_poses, n_kept);
  if (rc) {
    *n_poses = 0;
    return rc;
  }
  madicp_deskew_poses(T_prev, T_now, sensor_hz, *n_poses, poses);
  return MADICP_OK;
}

// theta = atan2(sq, half_b) / 3, cos, sin for n nodes (eig3.h): the libm calls of the device-side tree build,
// evaluated by the host's glibc so that the trees are the reference's bit for bit.
void madicp_host_trig(const double* args, double* res, int n, int num_threads) {
  const int threads = (n < 512 || num_threads < 2) ? 1 : (num_threads > 64 ? 64 : num_threads);
  for_chunks(threads, size_t(n), 256, [&](size_t c0, size_t c1) {
    for (size_t j = c0; j < c1; ++j) {
      const double theta = std::atan2(args[2 * j], args[2 * j + 1]) * (1.0 / 3.0);
      res[2 * j] = std::cos(theta);
      res[2 * j + 1] = std::sin(theta);
    }
  });
}

// > 0 while a device build strings its per-level libm sections together: the pool's workers keep spinning between them
void madicp_host_hot(int on) { madicp_host::g_hot.fetch_add(on ? 1 : -1, std::memory_order_relaxed); }

void madicp_host_for(int n, int num_threads, const std::function<void(int)>& fn) {
  for_chunks(std::max(1, std::min(num_threads, 64)), size_t(n), 1, [&](size_t c0, size_t c1) {
    for (size_t i = c0; i < c1; ++i) fn(int(i));
  });
}

// Diagnostic: sorts n pseudo-random keys drawn from `distinct` values (many ties when distinct << n) with
// std::sort and with the parallel restatement; returns the number of positions where the permutations differ.
extern "C" int64_t madicp_debug_sort_check(int64_t n, uint32_t seed, int64_t distinct, int num_threads) {
  if (n < 0 || distinct < 1) return -1;
  std::vector<Item> a(static_cast<size_t>(n)), b2;
  uint64_t st = seed * 0x9E3779B97F4A7C15ull + 0x1234567ull;
  for (int64_t i = 0; i < n; ++i) {
    st = st * 6364136223846793005ull + 1442695040888963407ull;
    a[size_t(i)] = Item{double((st >> 33) % uint64_t(distinct)) * 0.37 - 1.0, int32_t(i), 0};
  }
  b2 = a;
  std::sort(a.begin(), a.end(), KeyLess());
  sort_like_std(b2.data(), b2.data() + b2.size(), num_threads < 1 ? 1 : num_threads);
  int64_t diff = 0;
  for (int64_t i = 0; i < n; ++i) diff += (a[size_t(i)].idx != b2[size_t(i)].idx);
  return diff;
}

// Diagnostic: the deskew plan of a scan of records on the host, either as the order half on the calling thread alone
// followed by the pose half (split != 0: what a look-ahead plan does) or as madicp_deskew_plan on num_threads threads
// (split == 0: what the ingest does).  perm / chunk: desc->n entries; poses: 1024 x 12.
extern "C" int madicp_debug_deskew_plan(const madicp_points_t* desc, const madicp_vcorr_t* vcorr, const double T_prev[12],
                                        const double T_now[12], double sensor_hz, int split, int num_threads, int32_t* perm,
                                        uint16_t* chunk, double* poses, int* n_poses, int64_t* n_kept) {
  if (int e = madicp::check_points(desc, "madicp_debug_deskew_plan")) return e;
  if (int e = madicp::check_vcorr(vcorr, "madicp_debug_deskew_plan")) return e;
  if (!T_prev || !T_now || !(sensor_hz > 0.0) || !perm || !chunk || !poses || !n_poses || !n_kept) {
    madicp::set_error("madicp_debug_deskew_plan: bad arguments");
    return MADICP_ERR_INVALID;
  }
  madicp::VcorrTable table;
  const madicp_vcorr_t v = madicp::vcorr_of(vcorr);
  if (v.enabled) madicp::vcorr_table_fill(v.angle, &table);
  const madicp::VcorrTable* vt = v.enabled ? &table : nullptr;
  int rc = MADICP_OK;
  if (!split) {
    rc = madicp_deskew_plan(*desc, vt, T_prev, T_now, sensor_hz, num_threads, perm, chunk, poses, n_poses, n_kept);
  } else {
    rc = madicp_deskew_order(*desc, vt, 1, perm, chunk, n_poses, n_kept);
    if (!rc) madicp_deskew_poses(T_prev, T_now, sensor_hz, *n_poses, poses);
  }
  if (rc == MADICP_ERR_STATE)
    madicp::set_error("madicp_debug_deskew_plan: a point's rotation angle lies outside the table of the vertical correction");
  return rc;
}

// The deskew by time stamps on the host (time_deskew.h): the gate, the correction's table check, the default t_end (the
// largest kept stamp) and the chunk of every kept point, in record order.
extern "C" int madicp_debug_time_chunks(const madicp_points_t* desc, const madicp_vcorr_t* vcorr, const madicp_times_t* times,
                                        double sensor_hz, uint16_t* chunk_out, int64_t* n_kept) {
  const char* fn = "madicp_debug_time_chunks";
  if (int e = madicp::check_points(desc, fn)) return e;
  if (int e = madicp::check_vcorr(vcorr, fn)) return e;
  if (int e = madicp::check_times(times, desc, fn)) return e;
  if (!times || times->type == madicp::kTimeNone || !(sensor_hz > 0.0) || !std::isfinite(sensor_hz) || !chunk_out || !n_kept) {
    madicp::set_error(std::string(fn) + ": bad arguments (a time field, a finite rate > 0, outputs)");
    return MADICP_ERR_INVALID;
  }
  const madicp_times_t tm = madicp::times_of(times);
  madicp::VcorrTable table;
  const madicp_vcorr_t v = madicp::vcorr_of(vcorr);
  if (v.enabled) madicp::vcorr_table_fill(v.angle, &table);
  std::vector<double> tau;
  tau.reserve(size_t(desc->n));
  bool bad_angle = false, bad_time = false;
  unsigned long long tmax = 0;
  auto run = [&](auto zero) {
    const madicp::RecReader<decltype(zero)> rd(*desc, v.enabled ? &table : nullptr);
    for (int64_t i = 0; i < desc->n; ++i) {
      double x, y, z;
      if (!rd.kept_point(i, x, y, z, bad_angle)) continue;
      const double t = madicp::time_at(*desc, tm, i);
      if (std::isfinite(t)) tmax = std::max(tmax, madicp::time_key(t));
      else bad_time = true;
      tau.push_back(t);
    }
  };
  if (desc->is_f32) run(0.0f);
  else run(0.0);
  if (bad_angle || bad_time) {
    madicp::set_error(std::string(fn) + (bad_time ? ": a kept point's time stamp is NaN or infinite"
                                                   : ": a point's rotation angle lies outside the table of the vertical correction"));
    return MADICP_ERR_STATE;
  }
  const double t_end = tm.has_t_end ? tm.t_end : madicp::time_of_key(tmax);
  for (size_t i = 0; i < tau.size(); ++i) chunk_out[i] = uint16_t(madicp::time_chunk(tau[i], t_end, tm.scale, sensor_hz));
  *n_kept = int64_t(tau.size());
  return MADICP_OK;
}

extern "C" int madicp_debug_chunk_poses(const double T_prev[12], const double T_now[12], double sensor_hz, int n_chunks,
                                        double* poses) {
  if (!T_prev || !T_now || !(sensor_hz > 0.0) || n_chunks < 0 || n_chunks > 65536 || (n_chunks && !poses)) {
    madicp::set_error("madicp_debug_chunk_poses: bad arguments");
    return MADICP_ERR_INVALID;
  }
  madicp_deskew_poses(T_prev, T_now, sensor_hz, n_chunks, poses);
  return MADICP_OK;
}
