// pipeline.hpp -- the per-scan odometry driver with the reference's interface (odometry/pipeline.h:45-103),
// host C++, calling the GPU registration through the facade.  What it does per scan is the reference's
// Pipeline::compute (odometry/pipeline.cpp:125-265): optional deskew, MAD-tree of the scan, constant-
// velocity prediction, the ICP loop (one persistent-kernel launch instead of 15 OpenMP rounds), inlier
// ratio, velocity smoothing (odometry/vel_estimator.cpp), frame weight det(H^-1), keyframe promotion.
// How it is organised differs: by default the scan never exists as a tree on the host -- it is ingested (float
// conversion, deskew) and its MAD-tree is built ON THE DEVICE, its leaves become the moving leaves there, and on
// promotion the tree is transformed and laid out in a keyframe slot there (MADICP_GPU_BUILD=0: host-built flat
// trees, uploaded at promotion); the small dense algebra uses plain row-major arrays.
#pragma once
#include <algorithm>
#include <chrono>
#include <cstdlib>
#include <deque>
#include <limits>

#include "../pose_math.h"
#include "../records.hpp"
#include "facade.hpp"

namespace madicp_b200 {
// A scan whose records are device memory (a CUDA tensor, a CuPy array): read in place by the _dev entry points, after the
// context's stream waits for `stream`, the stream they are written on (0: the legacy default stream)
struct DevScan {
  void* stream = nullptr;
};
namespace detail {

using madicp_pose::Pose;
using madicp_pose::poseIdentity;
using madicp_pose::poseMul;
using madicp_pose::poseInverse;
using madicp_pose::poseFromTwist;
using madicp_pose::logSO3;
inline Vector3d poseApply(const Pose& T, const Vector3d& p) {
  Vector3d o;
  madicp_pose::poseApply(T, p.data(), o.data());
  return o;
}
// 1 / det(H) by partial-pivot LU (odometry/pipeline.cpp:223: H.inverse().determinant())
inline double inverseDeterminant(const double H[36]) {
  double A[36];
  std::memcpy(A, H, sizeof(A));
  double det = 1.0;
  for (int k = 0; k < 6; ++k) {
    int p = k;
    for (int i = k + 1; i < 6; ++i)
      if (std::fabs(A[i * 6 + k]) > std::fabs(A[p * 6 + k])) p = i;
    if (p != k) {
      for (int c = 0; c < 6; ++c) std::swap(A[k * 6 + c], A[p * 6 + c]);
      det = -det;
    }
    det *= A[k * 6 + k];
    for (int i = k + 1; i < 6; ++i) {
      const double f = A[i * 6 + k] / A[k * 6 + k];
      for (int c = k; c < 6; ++c) A[i * 6 + c] -= f * A[k * 6 + c];
    }
  }
  // a zero last pivot gives NaN, as the reference's inverse().determinant() does (solve6.h inv_det6)
  return (A[35] == 0.0) ? std::numeric_limits<double>::quiet_NaN() : 1.0 / det;
}

// odometry/vel_estimator.cpp:45-97.  J = I*dt makes H diagonal, so the 6x6 LDLT of the reference reduces to
// six independent divisions (with the same zero-pivot rule: a zero diagonal gives a zero update).
struct VelocityEstimator {
  double X[6] = {0, 0, 0, 0, 0, 0};
  double ts;
  explicit VelocityEstimator(double hz) : ts(1. / hz) {}
  void oneRound(const std::vector<Pose>& odom) {
    double Hd[6] = {0, 0, 0, 0, 0, 0}, b[6] = {0, 0, 0, 0, 0, 0};
    const Pose& now = odom.back();
    for (size_t i = 0; i + 1 < odom.size(); ++i) {
      const double dt = (odom.size() - 1 - i) * ts;
      const double weight = 1.f - double(odom.size() - 2 - i) / double(odom.size() - 1);
      const Pose T = poseMul(poseInverse(odom[i]), now);
      double e[6];
      for (int a = 0; a < 3; ++a) e[a] = dt * X[a] - T.m[a * 4 + 3];
      e[3] = dt * X[3] - std::atan2(-T.m[6], T.m[10]);
      e[4] = dt * X[4] - std::asin(T.m[2]);
      e[5] = dt * X[5] - std::atan2(-T.m[1], T.m[0]);
      double chi2 = 0;
      for (int a = 0; a < 6; ++a) chi2 += e[a] * e[a];
      const double chi = std::sqrt(chi2);
      const double sw = ((chi > 0.3162) ? 0.3162 / chi : 1.) * weight;
      for (int a = 0; a < 6; ++a) {
        Hd[a] += (sw * dt) * dt;
        b[a] += (sw * dt) * e[a];
      }
    }
    for (int a = 0; a < 6; ++a)
      if (std::fabs(Hd[a]) > std::numeric_limits<double>::min()) X[a] += -b[a] / Hd[a];
  }
};
}  // namespace detail

// Look-ahead tree builds: scans handed to Pipeline::prefetch are queued; when compute() needs the tree of the oldest
// one, the trees of ALL queued scans (up to `batch`) are built in one go, as one forest (madtree_gpu_build_batch) --
// the build's latency is that of its dependent-add chains, which a batch runs side by side -- and compute() then
// consumes them in FIFO order.  Possible because a scan's tree depends on the pose estimates only when the scan is
// deskewed (pipeline.cpp:137-141).  No threads: the batch is built by the thread that calls compute().
// A deskewed scan queues a plan instead (madicp_plan_points, pushPlan): its records go up and the pose-free half of its
// deskew (gate, correction, azimuth sort, chunks) runs on a library thread at once; compute() then consumes it with
// the latest poses (madicp_ingest_plan) and builds its tree alone -- the tree depends on the poses of the scan before.
class Lookahead {
 public:
  struct Job {
    std::vector<double> f64;  // private copies of the cloud ...
    std::vector<float> f32;
    const void* ext = nullptr;        // ... or the caller's buffer, kept alive by `keepalive` until its tree is built
    bool is_f32 = false;
    bool records = false;             // raw sensor records (Pipeline::prefetchRecords): `pts` describes them, `vc` is
    madicp_points_t pts{};            // their vertical correction (disabled: none)
    madicp_vcorr_t vc{};
    bool dev = false;                 // records in device memory, ready on `stream` (DevScan): never staged
    void* stream = nullptr;
    std::shared_ptr<void> keepalive;
    size_t n = 0;
    madtree_gpu_t* tree = nullptr;
    madicp_plan_t* plan = nullptr;  // a deskewed scan's look-ahead plan (pushPlan)
    const void* data() const { return ext ? ext : (is_f32 ? static_cast<const void*>(f32.data()) : static_cast<const void*>(f64.data())); }
  };
  Lookahead(madicp_ctx_t* ctx, double b_max, double b_min, int batch) : ctx_(ctx), b_max_(b_max), b_min_(b_min), batch_(batch) {}
  ~Lookahead() {
    madicp_stage_discard(ctx_);  // uploads and background sums may still be reading the queued clouds
    for (auto& j : fifo_) {
      if (j.tree) madtree_gpu_free(j.tree);
      if (j.plan) madicp_plan_free(j.plan);  // (returns once nothing reads the scan's buffer)
    }
  }
  void push(Job&& j) {
    fifo_.push_back(std::move(j));
    stageQueued();
  }
  // a deskewed scan: planned at once, over its records or its packed cloud, with at most num_threads plans' order
  // halves running at a time
  void pushPlan(Job&& j, int num_threads) {
    fifo_.push_back(std::move(j));
    Job& q = fifo_.back();  // (planned where its private copy, if any, will stay)
    const madicp_points_t d = q.records ? q.pts : madicp::packed_points(q.data(), int64_t(q.n), q.is_f32 ? 1 : 0);
    const int rc = q.dev ? madicp_plan_points_dev(ctx_, &d, &q.vc, num_threads, q.stream, &q.plan)
                         : madicp_plan_points(ctx_, &d, q.records ? &q.vc : nullptr, num_threads, &q.plan);
    if (rc < 0) {
      const std::string msg = "madicp_plan_points failed (" + std::to_string(rc) + "): " + madicp_last_error();
      fifo_.pop_back();
      throw Error(msg);
    }
  }
  bool empty() const { return fifo_.empty(); }
  size_t size() const { return fifo_.size(); }
  bool frontIsPlan() const { return !fifo_.empty() && fifo_.front().plan; }
  // the oldest queued scan, a planned one (the caller consumes the plan)
  Job popPlan() {
    Job j = std::move(fifo_.front());
    fifo_.pop_front();
    return j;
  }
  // tree of the oldest prefetched scan
  madtree_gpu_t* pop() {
    if (!fifo_.front().tree) buildBatch();
    madtree_gpu_t* t = fifo_.front().tree;
    fifo_.front().tree = nullptr;
    fifo_.pop_front();
    --built_;
    return t;
  }

 private:
  // scans that can share one batch call: packed clouds of one element type, or records (each with its own correction:
  // the batch call takes one per scan) -- host records, or device records ready on one stream
  static bool sameKind(const Job& a, const Job& b) {
    return !a.plan && !b.plan && a.records == b.records && (a.records || a.is_f32 == b.is_f32) && a.dev == b.dev &&
           (!a.dev || a.stream == b.stream);
  }
  // Builds the trees of the longest run of queued scans of the front's kind, up to the batch size.  A scan whose tree
  // cannot be built (records the range gate leaves empty) fails the batch call as a whole: the run is then halved until
  // the batch no longer contains it, and once the front scan fails on its own it is dropped from the queue and its
  // error is raised -- in the compute() call that reaches that scan.  The scans after it stay queued.
  void buildBatch() {
    size_t k = 0;
    const Job& front = fifo_.front();
    for (const Job& j : fifo_) {
      if (int(k) == batch_ || j.tree || !sameKind(j, front)) break;
      ++k;
    }
    std::vector<madtree_gpu_t*> out;
    for (;;) {
      std::vector<const void*> ptr;
      std::vector<int64_t> n;
      std::vector<madicp_points_t> pts;
      std::vector<madicp_vcorr_t> vc;
      for (size_t i = 0; i < k; ++i) {
        ptr.push_back(fifo_[i].data());
        n.push_back(int64_t(fifo_[i].n));
        pts.push_back(fifo_[i].pts);
        vc.push_back(fifo_[i].vc);
      }
      out.assign(k, nullptr);
      const int rc =
          front.dev ? madtree_gpu_build_batch_points_dev(ctx_, pts.data(), vc.data(), int(k), b_max_, b_min_, front.stream,
                                                         out.data())
          : front.records ? madtree_gpu_build_batch_points_ex(ctx_, pts.data(), vc.data(), int(k), b_max_, b_min_, out.data())
                          : madtree_gpu_build_batch(ctx_, ptr.data(), n.data(), front.is_f32 ? 1 : 0, int(k), b_max_, b_min_,
                                                    out.data());
      if (rc >= 0) break;
      const std::string msg = std::string(front.records ? "madtree_gpu_build_batch_points" : "madtree_gpu_build_batch") +
                              " failed (" + std::to_string(rc) + "): " + madicp_last_error();
      madicp_stage_discard(ctx_);  // (the failed call consumed the early uploads, or they are given up here)
      staged_ = 0;
      if (k == 1) {
        fifo_.pop_front();
        stageQueued();
        throw Error(msg);
      }
      k /= 2;
    }
    built_ = out.size();
    staged_ = 0;  // (the batch call consumed or discarded every early upload)
    for (size_t i = 0; i < out.size(); ++i) {
      Job& j = fifo_[i];
      j.tree = out[i];
      j.keepalive.reset();  // (the clouds have been copied to the device: pageable copies are staged before the call returns)
      j.f64 = std::vector<double>();
      j.f32 = std::vector<float>();
    }
    stageQueued();
  }
  // Early upload (madicp_stage_cloud) of the queued scans whose trees are not built yet, oldest first, up to one
  // batch: the copies run while the device registers the scans before them.
  void stageQueued() {
    while (staged_ < size_t(batch_) && built_ + staged_ < fifo_.size()) {
      const Job& j = fifo_[built_ + staged_];
      if (j.plan || j.dev || !sameKind(j, fifo_[built_])) break;
      if (j.records)
        check(madicp_stage_points_ex(ctx_, &j.pts, &j.vc, int64_t(batch_) * int64_t(j.n)), "madicp_stage_points");
      else
        check(madicp_stage_cloud(ctx_, j.data(), int64_t(j.n), j.is_f32 ? 1 : 0, int64_t(batch_) * int64_t(j.n)),
              "madicp_stage_cloud");
      ++staged_;
    }
  }
  madicp_ctx_t* ctx_;
  double b_max_, b_min_;
  int batch_;
  size_t built_ = 0, staged_ = 0;  // the first built_ queued scans have their trees; the next staged_ are on their way up
  std::deque<Job> fifo_;
};

class Pipeline {
 public:
  static constexpr int kMaxIcpIts = 15, kSmoothingT = 10, kFrameWindow = 10, kChunks = 1024;  // tools/constants.h

  Pipeline(double sensor_hz, bool deskew, double b_max, double rho_ker, double p_th, double b_min, double b_ratio,
           int num_keyframes, int num_threads, bool realtime, int device = -1)
      : sensor_hz_(sensor_hz), deskew_(deskew), b_max_(b_max), p_th_(p_th), b_min_(b_min), num_keyframes_(num_keyframes),
        realtime_(realtime), icp_(b_max, rho_ker, b_ratio, num_threads, resolveDevice(device), std::max(num_keyframes, 1)),
        vel_(sensor_hz) {
    frame_to_map_ = keyframe_to_map_ = detail::poseIdentity();
    if (const char* e = std::getenv("MADICP_GPU_BUILD")) gpu_build_ = std::atoi(e) != 0;
    num_threads_ = std::max(num_threads, 1);
    int lvl = 0;
    while ((1 << (lvl + 1)) <= std::max(num_threads, 1)) ++lvl;
    max_parallel_levels_ = lvl;  // pipeline.cpp:64
    timing_ = std::getenv("MADICP_PIPELINE_TIMING") != nullptr;
  }
  ~Pipeline() {
    if (timing_ && timed_scans_ > 0)
      std::fprintf(stderr, "Pipeline phases, mean over %d scans [ms]: deskew %.3f  tree build %.3f  set moving %.3f  "
                   "register (incl. keyframe upload) %.3f  rest %.3f  | prefetch (outside compute) %.3f\n", timed_scans_,
                   t_ph_[0] / timed_scans_, t_ph_[1] / timed_scans_, t_ph_[2] / timed_scans_, t_ph_[3] / timed_scans_,
                   t_ph_[4] / timed_scans_, t_prefetch_ / timed_scans_);
  }

  // the reference's constructor has no device argument: MADICP_DEVICE selects the GPU (default 0)
  static int resolveDevice(int device) {
    if (device >= 0) return device;
    const char* e = std::getenv("MADICP_DEVICE");
    return e ? std::atoi(e) : 0;
  }
  Matrix4d currentPose() const { return toM(frame_to_map_); }
  std::vector<Matrix4d> trajectory() const {
    std::vector<Matrix4d> out;
    for (const auto& p : trajectory_) out.push_back(toM(p));
    return out;
  }
  Matrix4d keyframePose() const { return toM(keyframe_to_map_); }
  bool isInitialized() const { return is_initialized_; }
  bool isMapUpdated() const { return is_map_updated_; }
  size_t currentID() const { return seq_; }
  size_t keyframeID() const { return seq_keyframe_; }
  double inliersRatio() const { return inliers_ratio_; }
  size_t numKeyframes() const { return keyframes_.size(); }
  ContainerType currentLeaves() const { return current_ ? current_->tree->leafMeans() : ContainerType(); }
  ContainerType modelLeaves() const {
    ContainerType all;
    for (const auto& f : keyframes_) {
      ContainerType l = f->tree->leafMeans();
      all.insert(all.end(), l.begin(), l.end());
    }
    return all;
  }

  // test hook: the deskew step alone (poses 4x4 row-major)
  static ContainerType deskewOnly(ContainerType cloud, const Matrix4d& T_prev, const Matrix4d& T_now, double sensor_hz,
                                  int num_threads = 1) {
    detail::Pose a, b;
    std::memcpy(a.m, T_prev.m, sizeof(a.m));
    std::memcpy(b.m, T_now.m, sizeof(b.m));
    deskew(cloud, a, b, sensor_hz, num_threads);
    return cloud;
  }

  // pipeline.cpp:125-265; reference signature (pipeline.h:71): the cloud by value
  void compute(double stamp, ContainerType cloud) {
    if (cloud.empty()) throw Error("Pipeline.compute: empty cloud");
    computeRaw(stamp, cloud[0].data(), cloud.size(), false);
  }
  // the same without taking ownership: N x 3 doubles read in place
  void compute(double stamp, const double* xyz, size_t n) { computeRaw(stamp, xyz, n, false); }
  // float32 scans as the dataset readers produce them (the conversion to float64 runs on the device)
  void computeF32(double stamp, const float* xyz, size_t n) {
    if (!gpu_build_) {
      ContainerType cloud(n);
      for (size_t i = 0; i < n; ++i)
        for (int a = 0; a < 3; ++a) cloud[i][size_t(a)] = double(xyz[3 * i + size_t(a)]);
      compute(stamp, std::move(cloud));
      return;
    }
    computeRaw(stamp, xyz, n, true);
  }
  // Raw sensor records with the dataset readers' range gate (include/madicp_b200.h, madicp_points_t), read in place:
  // the same result as compute() on the reader's filtered array -- corrected by `vc` (nullable: none) like KITTI's
  // reader with apply_correction.  MADICP_GPU_BUILD=0: the kept points are packed (and corrected) on the host with the
  // same restatement, then the host path runs.
  // dev (nullable): the records are device memory, read in place (host-built trees, MADICP_GPU_BUILD=0, need host records:
  // the caller copies them over first)
  void computeRecords(double stamp, const madicp_points_t& pts, const madicp_vcorr_t* vc = nullptr, const DevScan* dev = nullptr) {
    check(madicp::check_vcorr(vc, "Pipeline.computeRecords"), "Pipeline.computeRecords");
    if (dev && !gpu_build_) throw Error("Pipeline.computeRecords: device records need device-built trees (MADICP_GPU_BUILD)");
    if (!gpu_build_) {
      compute(stamp, packRecords(pts, vc));
      return;
    }
    if (!pts.data || pts.n <= 0) throw Error("Pipeline.computeRecords: empty scan");
    const madicp_vcorr_t v = madicp::vcorr_of(vc);
    computeRaw(stamp, pts.data, size_t(pts.n), pts.is_f32 != 0, &pts, &v, dev);
  }
  bool gpuBuild() const { return gpu_build_; }
  int lastIcpIterations() const { return last_iters_; }  // rounds the realtime budget allowed for the last scan
  // Hands a FUTURE scan over for a look-ahead (batched) tree build (see Lookahead).  compute() then consumes the
  // prefetched scans in the order they were handed over and ignores its own cloud argument for them.  Returns false (and does
  // nothing) when look-ahead is not possible: host-built trees, or deskewing without deskew_ahead (the scan needs the
  // latest poses).  deskew_ahead on a deskewing pipeline: the scan is planned instead -- uploaded, gated, corrected and
  // sorted by azimuth ahead of time; compute() applies the chunk poses and builds its tree (no effect without deskew).
  // keepalive: when given, the buffer is read in place (no copy) and the handle is dropped once compute() has consumed
  // the scan; without it the cloud is copied.
  // dev (nullable, records only): the records are device memory (DevScan), kept alive until their tree is built or their
  // plan consumed.
  bool prefetch(const void* xyz, size_t n, bool is_f32, std::shared_ptr<void> keepalive = nullptr,
                const madicp_points_t* records = nullptr, const madicp_vcorr_t* vc = nullptr, bool deskew_ahead = false,
                const DevScan* dev = nullptr) {
    if (!gpu_build_ || (deskew_ && !deskew_ahead) || !xyz || n == 0) return false;
    const auto p0 = clk();
    struct Tick {  // (the hand-over runs on the thread that launches the registrations: its cost is part of the scan's)
      Pipeline* p; std::chrono::steady_clock::time_point t0;
      ~Tick() { if (p->timing_) p->t_prefetch_ += ms(t0, clk()); }
    } tick{this, p0};
    if (!lookahead_) {
      int batch = 32;
      if (const char* e = std::getenv("MADICP_LOOKAHEAD")) batch = std::atoi(e);
      if (batch < 1) return false;
      lookahead_.reset(new Lookahead(icp_.context(), b_max_, b_min_, std::min(batch, 64)));
    }
    Lookahead::Job j;
    j.n = n;
    j.is_f32 = is_f32;
    if (records) {  // (read in place: the caller must hand over a keepalive)
      if (!keepalive) throw Error("Pipeline.prefetchRecords: the records must be kept alive");
      // a descriptor the library would reject must not enter the queue (every later batch would fail on it)
      check(madicp::check_points(records, "Pipeline.prefetchRecords"), "Pipeline.prefetchRecords");
      check(madicp::check_vcorr(vc, "Pipeline.prefetchRecords"), "Pipeline.prefetchRecords");
      j.records = true;
      j.pts = *records;
      j.vc = madicp::vcorr_of(vc);
      j.dev = dev != nullptr;
      j.stream = dev ? dev->stream : nullptr;
    }
    if (keepalive) {
      j.ext = xyz;
      j.keepalive = std::move(keepalive);
    } else if (is_f32) {
      j.f32.assign(static_cast<const float*>(xyz), static_cast<const float*>(xyz) + 3 * n);
    } else {
      j.f64.assign(static_cast<const double*>(xyz), static_cast<const double*>(xyz) + 3 * n);
    }
    if (deskew_) lookahead_->pushPlan(std::move(j), num_threads_);
    else lookahead_->push(std::move(j));
    return true;
  }
  bool prefetchRecords(const madicp_points_t& pts, std::shared_ptr<void> keepalive, const madicp_vcorr_t* vc = nullptr,
                       bool deskew_ahead = false, const DevScan* dev = nullptr) {
    return prefetch(pts.data, pts.n > 0 ? size_t(pts.n) : 0, pts.is_f32 != 0, std::move(keepalive), &pts, vc, deskew_ahead,
                    dev);
  }
  size_t prefetched() { return lookahead_ ? lookahead_->size() : 0; }

 private:
  // the scan's MAD-tree: ingest (+ deskew, pipeline.cpp:137-138) and build, on the device or on the host
  std::unique_ptr<MADtree> makeTree(const void* xyz, size_t n, bool is_f32, const madicp_points_t* records,
                                    const madicp_vcorr_t* vc, const DevScan* dev) {
    const bool dsk = deskew_ && is_initialized_ && trajectory_.size() > 1;
    const double* Ta = dsk ? trajectory_[trajectory_.size() - 2].m : nullptr;
    const double* Tb = dsk ? trajectory_[trajectory_.size() - 1].m : nullptr;
    if (lookahead_ && lookahead_->frontIsPlan()) {  // planned ahead of time: the chunk poses, the ingest, the tree
      const Lookahead::Job j = lookahead_->popPlan();  // (a failure leaves the scans after it queued)
      check(madicp_ingest_plan(icp_.context(), j.plan, dsk ? 1 : 0, Ta, Tb, sensor_hz_, nullptr, nullptr), "madicp_ingest_plan");
      return std::unique_ptr<MADtree>(new MADtree(icp_.context(), b_max_, b_min_));
    }
    if (lookahead_ && !lookahead_->empty())  // built ahead of time by a worker lane
      return std::unique_ptr<MADtree>(new MADtree(icp_.context(), lookahead_->pop(), b_max_));
    if (gpu_build_ && records && dev) {
      check(madicp_ingest_points_dev(icp_.context(), records, vc, dsk ? 1 : 0, Ta, Tb, sensor_hz_,
                                     std::max(1 << max_parallel_levels_, 1), dev->stream, nullptr, nullptr),
            "madicp_ingest_points_dev");
      return std::unique_ptr<MADtree>(new MADtree(icp_.context(), b_max_, b_min_));
    }
    if (gpu_build_ && records) {
      check(madicp_ingest_points_ex(icp_.context(), records, vc, dsk ? 1 : 0, Ta, Tb, sensor_hz_,
                                    std::max(1 << max_parallel_levels_, 1), nullptr, nullptr), "madicp_ingest_points");
      return std::unique_ptr<MADtree>(new MADtree(icp_.context(), b_max_, b_min_));
    }
    if (gpu_build_) {
      check(madicp_ingest(icp_.context(), xyz, int64_t(n), is_f32 ? 1 : 0, dsk ? 1 : 0, Ta, Tb, sensor_hz_,
                          std::max(1 << max_parallel_levels_, 1), nullptr), "madicp_ingest");
      return std::unique_ptr<MADtree>(new MADtree(icp_.context(), b_max_, b_min_));
    }
    const double* pts = static_cast<const double*>(xyz);
    if (dsk) {
      ContainerType cloud(n);
      std::memcpy(cloud[0].data(), pts, sizeof(double) * 3 * n);
      check(madicp_deskew(cloud[0].data(), int64_t(n), Ta, Tb, sensor_hz_, 1 << max_parallel_levels_), "madicp_deskew");
      return std::unique_ptr<MADtree>(new MADtree(cloud[0].data(), n, b_max_, b_min_, max_parallel_levels_));
    }
    return std::unique_ptr<MADtree>(new MADtree(pts, n, b_max_, b_min_, max_parallel_levels_));
  }

  void computeRaw(double stamp, const void* xyz, size_t n, bool is_f32, const madicp_points_t* records = nullptr,
                  const madicp_vcorr_t* vc = nullptr, const DevScan* dev = nullptr) {
    if (!xyz || n == 0) throw Error("Pipeline.compute: empty cloud");
    is_map_updated_ = false;
    if (!is_initialized_) {  // pipeline.cpp:267-284
      auto f = std::make_shared<FrameB>();
      f->frame = int(seq_);
      f->to_map = frame_to_map_;
      f->stamp = stamp;
      f->tree = makeTree(xyz, n, is_f32, records, vc, dev);
      keyframes_.push_back(f);
      current_ = f;
      trajectory_.push_back(detail::poseIdentity());
      is_initialized_ = is_map_updated_ = true;
      ++seq_;
      return;
    }
    const auto c0 = clk();
    const auto c1 = c0;
    auto cur = std::make_shared<FrameB>();
    cur->tree = makeTree(xyz, n, is_f32, records, vc, dev);
    const auto c2 = clk();
    double t[3], w[3];
    for (int a = 0; a < 3; ++a) {
      t[a] = vel_.X[a] * 1. / sensor_hz_;
      w[a] = vel_.X[3 + a] * 1. / sensor_hz_;
    }
    const detail::Pose prediction = detail::poseMul(frame_to_map_, detail::poseFromTwist(t, w));
    icp_.setMoving(*cur->tree);
    const auto c3 = clk();
    icp_.init(toM(prediction));
    std::vector<const MADtree*> kfs;
    for (const auto& f : keyframes_) kfs.push_back(f->tree.get());
    // `realtime` (pipeline.cpp:62,167-169): round k runs only while preprocessing + the rounds so far + one more
    // round of the last duration still fit the sensor period minus 5 ms.  The rounds of a scan run in ONE launch
    // here, so the budget is turned into a round count up front, with the per-round time of the previous scan as
    // the duration of a round; a loop cut short keeps the union of the matched flags (no clear ever happened).
    int iters = kMaxIcpIts;
    if (realtime_) {
      const double budget = (1000.0 / sensor_hz_) - 5.0 - ms(c0, c3);
      if (budget < 0.0) iters = 0;
      else if (round_ms_ > 0.0) iters = std::max(1, std::min(kMaxIcpIts, int(std::floor(budget / round_ms_))));
    }
    last_iters_ = iters;
    const int matched = icp_.compute(kfs, iters, iters < kMaxIcpIts);  // the whole loop of pipeline.cpp:166-193
    const auto c4 = clk();
    if (iters > 0) round_ms_ = ms(c3, c4) / double(iters);
    std::memcpy(frame_to_map_.m, icp_.X_.m, sizeof(frame_to_map_.m));
    inliers_ratio_ = double(matched) / double(cur->tree->numLeaves());  // :197-204
    trajectory_.push_back(frame_to_map_);
    std::vector<detail::Pose> window;
    for (int i = std::max(0, int(trajectory_.size()) - kSmoothingT); i < int(trajectory_.size()); ++i)
      window.push_back(trajectory_[size_t(i)]);
    vel_.oneRound(window);  // :208-217
    cur->frame = int(seq_);
    cur->to_map = frame_to_map_;
    cur->stamp = stamp;
    cur->weight = (iters > 0 && iters <= MADICP_MAX_ITERS) ? icp_.weight()                        // :223, from the device
                                                           : detail::inverseDeterminant(icp_.H_adder_);
    cur->tree->applyTransform(toM(frame_to_map_));             // :224
    current_ = cur;
    frames_.push_back(cur);
    if (frames_.size() > size_t(kFrameWindow)) frames_.pop_front();
    if (inliers_ratio_ < p_th_) {  // :234-262
      double best_w = std::numeric_limits<double>::max();
      std::shared_ptr<FrameB> best;
      for (const auto& f : frames_)
        if (f->weight < best_w) {
          best_w = f->weight;
          best = f;
        }
      if (!best) best = cur;  // every weight inf/NaN (singular H): the reference dereferences null here; keep the newest
      while (!frames_.empty() && frames_.front()->frame <= best->frame) frames_.pop_front();
      keyframes_.push_back(best);
      if (keyframes_.size() > size_t(num_keyframes_)) keyframes_.pop_front();
      is_map_updated_ = true;
      seq_keyframe_ = size_t(best->frame);
      keyframe_to_map_ = best->to_map;
    }
    ++seq_;
    if (timing_) {
      const auto c5 = clk();
      t_ph_[0] += ms(c0, c1); t_ph_[1] += ms(c1, c2); t_ph_[2] += ms(c2, c3); t_ph_[3] += ms(c3, c4); t_ph_[4] += ms(c4, c5);
      ++timed_scans_;
    }
  }

  struct FrameB {  // tools/frame.h:37-51
    detail::Pose to_map;
    std::unique_ptr<MADtree> tree;
    double stamp = 0, weight = 0;
    int frame = 0;
  };
  static Matrix4d toM(const detail::Pose& p) {
    Matrix4d M = Matrix4d::Identity();
    std::memcpy(M.m, p.m, sizeof(p.m));
    return M;
  }
  // pipeline.cpp:79-123 on the host (madicp_deskew: threaded, same permutation and poses); the device path is
  // madicp_ingest
  static void deskew(ContainerType& cloud, const detail::Pose& T_prev, const detail::Pose& T_now, double sensor_hz,
                     int num_threads) {
    if (cloud.empty()) return;
    check(madicp_deskew(cloud[0].data(), int64_t(cloud.size()), T_prev.m, T_now.m, sensor_hz, num_threads), "madicp_deskew");
  }

  // the kept points of `pts` as a packed float64 cloud, corrected by `vc` (nullable), with the predicate and the
  // restatement the device applies (records.hpp)
  static ContainerType packRecords(const madicp_points_t& pts, const madicp_vcorr_t* vc) {
    check(madicp::check_points(&pts, "Pipeline.computeRecords"), "Pipeline.computeRecords");
    madicp::VcorrTable table;
    const bool corrected = madicp::vcorr_of(vc).enabled != 0;
    if (corrected) madicp::vcorr_table_fill(vc->angle, &table);
    ContainerType cloud;
    cloud.reserve(size_t(pts.n));
    bool bad = false;
    auto pack = [&](auto zero) {
      const madicp::RecReader<decltype(zero)> rd(pts, corrected ? &table : nullptr);
      for (int64_t i = 0; i < pts.n; ++i) {
        Vector3d p;
        if (rd.kept_point(i, p[0], p[1], p[2], bad)) cloud.push_back(p);
      }
    };
    if (pts.is_f32) pack(0.0f);
    else pack(0.0);
    if (bad) throw Error("Pipeline.computeRecords: a point's rotation angle lies outside the table of the vertical correction");
    if (cloud.empty()) throw Error("Pipeline.computeRecords: no point inside the range gate");
    return cloud;
  }

  static std::chrono::steady_clock::time_point clk() { return std::chrono::steady_clock::now(); }
  static double ms(std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) {
    return std::chrono::duration<double, std::milli>(b - a).count();
  }
  bool timing_ = false;  // MADICP_PIPELINE_TIMING: per-phase host wall clock, printed by the destructor
  int timed_scans_ = 0;
  double t_ph_[5] = {0, 0, 0, 0, 0}, t_prefetch_ = 0;
  double sensor_hz_;
  bool deskew_;
  double b_max_, p_th_, b_min_;
  int num_keyframes_, max_parallel_levels_ = 0;
  bool realtime_;
  bool gpu_build_ = true;   // MADICP_GPU_BUILD=0: host-built trees
  int num_threads_ = 1;
  int last_iters_ = 0;
  double round_ms_ = 0.0;   // duration of one GN round on the previous scan (realtime budget)
  MADicp icp_;
  std::unique_ptr<Lookahead> lookahead_;  // declared after icp_: destroyed first (its lanes use icp_'s context)
  detail::VelocityEstimator vel_;
  detail::Pose frame_to_map_, keyframe_to_map_;
  std::deque<std::shared_ptr<FrameB>> keyframes_, frames_;
  std::shared_ptr<FrameB> current_;
  std::vector<detail::Pose> trajectory_;
  size_t seq_ = 0, seq_keyframe_ = 0;
  bool is_initialized_ = false, is_map_updated_ = false;
  double inliers_ratio_ = 0;
};

}  // namespace madicp_b200
