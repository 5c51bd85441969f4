// facade.hpp -- C++ host facade over the C ABI (include/madicp_b200.h) that keeps the reference's
// class and method names, so code written against rvp-group/mad-icp's C++ API maps one to one:
//
//   reference (mad_icp/src)                              here (namespace madicp_b200)
//   tools/mad_tree.h        struct MADtree               class MADtree   (whole-tree handle, flat layout)
//   odometry/mad_icp.h      class MADicp                 class MADicp    (resetAdders/setMoving/init/update/
//                                                                         updateState + fused compute)
//   pybind/tools/mad_icp_wrapper.h   MADicpWrapper       class MADicpWrapper
//   pybind/tools/mad_tree_wrapper.h  MADtreeWrapper      class MADtreeWrapper
//
// Eigen is not required: vectors are std::array<double,3> (layout-compatible with Eigen::Vector3d, the
// same 24-byte stride the reference's buffer protocol relies on, pybind/eigen_stl_bindings.h:73-80) and
// poses are 4x4 row-major arrays.  With Eigen available, Eigen::Map<> over these buffers is zero-copy.
// All compute goes to the GPU through libmadicp_b200.so; nothing here falls back to the CPU.
#pragma once
#include <array>
#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <algorithm>
#include <memory>
#include <mutex>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../../include/madicp_b200.h"

namespace madicp_b200 {

using Vector3d = std::array<double, 3>;
using ContainerType = std::vector<Vector3d>;  // reference: tools/mad_tree.h:42
struct Matrix4d {                               // row-major 4x4
  double m[16];
  static Matrix4d Identity() {
    Matrix4d I{};
    I.m[0] = I.m[5] = I.m[10] = I.m[15] = 1.0;
    return I;
  }
};

struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};
inline void check(int rc, const char* what) {
  if (rc < 0) throw Error(std::string(what) + " failed (" + std::to_string(rc) + "): " + madicp_last_error());
}
inline void pose12(const Matrix4d& T, double X[12]) { std::memcpy(X, T.m, sizeof(double) * 12); }
inline Matrix4d from12(const double X[12]) {
  Matrix4d T = Matrix4d::Identity();
  std::memcpy(T.m, X, sizeof(double) * 12);
  return T;
}

// reference: struct MADtree (tools/mad_tree.h:47-102).  One object = one whole tree (the reference's
// root node); leaves are exposed as arrays in getLeafs (DFS) order instead of node pointers.  The tree lives
// either on the host (flat, built by madtree_build) or in the device memory of a registration context (built by
// the device builder from a cloud that madicp_ingest left there); both stay in the SENSOR frame: applyTransform
// records the pose, the device applies it when the tree is promoted to a keyframe, the host applies it to the
// leaf means it hands out.
class MADtree {
 public:
  // MADtree(vec, begin, end, b_max, b_min, 0, max_parallel_level, nullptr, nullptr) (mad_tree.cpp:33-45)
  MADtree(const ContainerType& cloud, double b_max, double b_min, int max_parallel_level = 0)
      : MADtree(cloud.empty() ? nullptr : cloud[0].data(), cloud.size(), b_max, b_min, max_parallel_level) {}
  // the same from a bare N x 3 buffer (the build copies the points into its own working memory)
  MADtree(const double* xyz, size_t n, double b_max, double b_min, int max_parallel_level = 0)
      : b_max_(b_max), uid_(next_uid()) {
    check(madtree_build(xyz, int64_t(n), b_max, b_min, 1 << (max_parallel_level > 0 ? max_parallel_level : 0), &t_),
          "madtree_build");
  }
  // built ON THE DEVICE from the cloud madicp_ingest left in `ctx` (tools/mad_tree.cpp:47-130, bit-identical)
  MADtree(madicp_ctx_t* ctx, double b_max, double b_min) : b_max_(b_max), uid_(next_uid()), ctx_(ctx) {
    check(madtree_gpu_build_resident(ctx, b_max, b_min, &g_), "madtree_gpu_build_resident");
  }
  // adopts a tree a build lane produced on `ctx`'s device (madicp_builder_build)
  MADtree(madicp_ctx_t* ctx, madtree_gpu_t* built, double b_max) : g_(built), b_max_(b_max), uid_(next_uid()), ctx_(ctx) {}
  ~MADtree() {
    madtree_free(t_);
    madtree_gpu_free(g_);
  }
  MADtree(const MADtree&) = delete;
  MADtree& operator=(const MADtree&) = delete;

  // reference: applyTransform(r, t) (mad_tree.cpp:165-172); T row-major 4x4.  The reference transforms every
  // scan's tree (pipeline.cpp:224) although only promoted frames are ever read again; here the pose is kept and
  // the transform (same arithmetic) runs on the device when the tree is uploaded as a keyframe.
  void applyTransform(const Matrix4d& T) {
    if (has_pose_) {  // a second transform: fold the first into the host tree (composing poses would round differently)
      if (!t_) throw Error("MADtree.applyTransform: a device-resident tree can be transformed once");
      check(madtree_apply_transform(t_, pose_), "madtree_apply_transform");
    }
    pose12(T, pose_);
    has_pose_ = true;
    ++version_;
  }
  int numLeaves() const { return t_ ? madtree_num_leaves(t_) : madtree_gpu_num_leaves(g_); }
  int numNodes() const { return t_ ? madtree_num_nodes(t_) : madtree_gpu_num_nodes(g_); }
  // reference: getLeafs(back_inserter) (mad_tree.cpp:154-163) -> leaf->mean_ (in the frame applyTransform put it in)
  ContainerType leafMeans() const { return leafMeans({this}); }
  // the same for several trees, tree after tree: sum(numLeaves) x 3 doubles
  static size_t numLeaves(const std::vector<const MADtree*>& trees) {
    size_t n = 0;
    for (const MADtree* t : trees) n += size_t(t->numLeaves());
    return n;
  }
  static ContainerType leafMeans(const std::vector<const MADtree*>& trees) {
    ContainerType out(numLeaves(trees));
    if (!out.empty()) leafMeans(trees, out[0].data());
    return out;
  }
  // Host output.  Device trees (one context) are gathered and posed on the device in one call; host-built trees are
  // read and posed here.
  static void leafMeans(const std::vector<const MADtree*>& trees, double* out) {
    if (!trees.empty() && trees[0]->g_) {
      std::vector<const madtree_gpu_t*> g;
      std::vector<const double*> X;
      deviceTable(trees, g, X);
      check(madtree_gpu_leaf_means(g.data(), X.data(), int(g.size()), out), "madtree_gpu_leaf_means");
      return;
    }
    for (const MADtree* t : trees) {
      if (!t->t_) throw Error("MADtree.leafMeans: host-built and device trees in one call");
      const size_t n = size_t(t->numLeaves());
      if (n == 0) continue;
      check(madtree_leaves(t->t_, out, nullptr, nullptr, nullptr), "madtree_leaves");
      if (t->has_pose_)
        for (size_t i = 0; i < n; ++i) {  // R*p + t, rows as (a*x + b*y) + c*z, translation last: the node transform's arithmetic
          double* p = out + 3 * i;
          const double x = p[0], y = p[1], z = p[2], *X = t->pose_;
          for (int r = 0; r < 3; ++r) p[r] = ((X[r * 4] * x + X[r * 4 + 1] * y) + X[r * 4 + 2] * z) + X[r * 4 + 3];
        }
      out += 3 * n;
    }
  }
  // Device output (device memory of the trees' device), ready on consumer_stream with no host sync; device trees only.
  static void leafMeansDev(const std::vector<const MADtree*>& trees, double* out, void* consumer_stream) {
    if (trees.empty()) return;
    std::vector<const madtree_gpu_t*> g;
    std::vector<const double*> X;
    deviceTable(trees, g, X);
    check(madtree_gpu_leaf_means_dev(g.data(), X.data(), int(g.size()), out, consumer_stream), "madtree_gpu_leaf_means_dev");
  }
  // The cloud the tree was built from, in the order the build got it, and the record index of every point
  // (madicp_set_keep_cloud for device trees; keepHostCloud for host-built ones).  posed: by the tree's pose, if any,
  // with the node transform's arithmetic; without a pose the points are copied untouched.
  size_t numCloudPoints() const {
    if (t_) {
      if (!host_cloud_) throw Error("MADtree.cloud: the tree kept no cloud");
      return host_idx_.size();
    }
    const int64_t n = madtree_gpu_num_cloud_points(g_);
    check(int(n < 0 ? n : 0), "madtree_gpu_num_cloud_points");
    return size_t(n);
  }
  // host output (xyz_out / idx_out nullable)
  void cloud(bool posed, double* xyz_out, int64_t* idx_out) const {
    const double* X = posed ? pose() : nullptr;
    if (g_) {
      check(int(std::min<int64_t>(0, madtree_gpu_cloud(g_, X, xyz_out, idx_out))), "madtree_gpu_cloud");
      return;
    }
    if (!host_cloud_) throw Error("MADtree.cloud: the tree kept no cloud");
    const size_t n = host_idx_.size();
    if (idx_out)
      for (size_t i = 0; i < n; ++i) idx_out[i] = host_idx_[i];
    if (!xyz_out) return;
    if (!X) {
      std::memcpy(xyz_out, host_xyz_.data(), n * 3 * sizeof(double));
      return;
    }
    for (size_t i = 0; i < n; ++i) {  // the node transform's arithmetic, as leafMeans
      const double* p = host_xyz_.data() + 3 * i;
      const double x = p[0], y = p[1], z = p[2];
      for (int r = 0; r < 3; ++r) xyz_out[3 * i + r] = ((X[r * 4] * x + X[r * 4 + 1] * y) + X[r * 4 + 2] * z) + X[r * 4 + 3];
    }
  }
  // device output (device memory of the tree's device), ready on consumer_stream with no host sync; device trees only
  void cloudDev(bool posed, double* xyz_out, int64_t* idx_out, void* consumer_stream) const {
    if (!g_) throw Error("MADtree.cloudDev: a device output needs a device tree");
    check(int(std::min<int64_t>(0, madtree_gpu_cloud_dev(g_, posed ? pose() : nullptr, xyz_out, idx_out, consumer_stream))),
          "madtree_gpu_cloud_dev");
  }
  // a host-built tree keeps `xyz` (n x 3) and its record indices
  void keepHostCloud(const double* xyz, size_t n, std::vector<int32_t> idx) {
    host_xyz_.assign(xyz, xyz + 3 * n);
    host_idx_ = std::move(idx);
    host_cloud_ = true;
  }
  void releaseCloud() {
    if (g_) madtree_gpu_release_cloud(g_);
    host_xyz_ = std::vector<double>();
    host_idx_ = std::vector<int32_t>();
    host_cloud_ = false;
  }
  const madtree_t* hostHandle() const { return t_; }
  const madtree_gpu_t* deviceHandle() const { return g_; }
  madicp_ctx_t* deviceContext() const { return ctx_; }
  const double* pose() const { return has_pose_ ? pose_ : nullptr; }
  double bMax() const { return b_max_; }
  // identity of the tree CONTENT for residency caches: unique per object (addresses get reused) and bumped
  // by every applyTransform
  uint64_t version() const { return (uid_ << 20) | version_; }

 private:
  static uint64_t next_uid() {
    static uint64_t counter = 0;
    return ++counter;
  }
  static void deviceTable(const std::vector<const MADtree*>& trees, std::vector<const madtree_gpu_t*>& g,
                          std::vector<const double*>& X) {
    for (const MADtree* t : trees) {
      if (!t->g_) throw Error("MADtree.leafMeans: a device gather needs device trees");
      g.push_back(t->g_);
      X.push_back(t->pose());
    }
  }
  madtree_t* t_ = nullptr;
  madtree_gpu_t* g_ = nullptr;
  double b_max_;
  uint64_t uid_;
  uint64_t version_ = 0;
  madicp_ctx_t* ctx_ = nullptr;
  bool has_pose_ = false;
  double pose_[12];
  bool host_cloud_ = false;  // keepHostCloud
  std::vector<double> host_xyz_;
  std::vector<int32_t> host_idx_;
};

// A voxel map of kept clouds on one context (madicp_map_*, not in the reference): owns the map and frees it.  Trees must be
// device trees of that context, built with madicp_set_keep_cloud on.
class VoxelMap {
 public:
  VoxelMap(madicp_ctx_t* ctx, double voxel_size, int points_per_voxel, int64_t reserve_points = 0) {
    check(madicp_map_create(ctx, voxel_size, points_per_voxel, reserve_points, &m_), "madicp_map_create");
  }
  ~VoxelMap() { madicp_map_free(m_); }
  VoxelMap(const VoxelMap&) = delete;
  VoxelMap& operator=(const VoxelMap&) = delete;

  // the tree's kept cloud, posed by its pose (none: untouched), its points tagged with `scan`
  void insert(const MADtree& t, int64_t scan) {
    if (!t.deviceHandle()) throw Error("VoxelMap.insert: the map takes device trees");
    check(int(std::min<int64_t>(0, madicp_map_insert(m_, t.deviceHandle(), t.pose(), scan))), "madicp_map_insert");
  }
  size_t size(int64_t* dropped = nullptr) {
    const int64_t n = madicp_map_size(m_, dropped);
    check(int(std::min<int64_t>(0, n)), "madicp_map_size");
    return size_t(n);
  }
  // host output (either nullable): size() x 3 doubles, size() x 2 int64 (scan, record)
  void points(double* xyz, int64_t* scan_record) {
    check(int(std::min<int64_t>(0, madicp_map_points(m_, xyz, scan_record))), "madicp_map_points");
  }
  // device output of the context's device, ready on consumer_stream with no host sync
  void pointsDev(double* xyz, int64_t* scan_record, void* consumer_stream) {
    check(int(std::min<int64_t>(0, madicp_map_points_dev(m_, xyz, scan_record, consumer_stream))), "madicp_map_points_dev");
  }
  void clear() { check(madicp_map_clear(m_), "madicp_map_clear"); }
  // every voxel whose centre lies farther than max_distance from origin goes, with its rows (asynchronous)
  void removeFar(const double origin[3], double max_distance) {
    check(madicp_map_remove_far(m_, origin, max_distance), "madicp_map_remove_far");
  }
  // the voxels the rays from the tree's pose (none: the origin) to its posed kept cloud pass through in their first
  // `reach` of steps go, with their rows, unless they hold one of its points (asynchronous)
  void carve(const MADtree& t, double reach) {
    if (!t.deviceHandle()) throw Error("VoxelMap.carve: the map takes device trees");
    check(madicp_map_carve(m_, t.deviceHandle(), t.pose(), reach), "madicp_map_carve");
  }
  // the nearest row within max_distance of each of n host queries (n x 3): row (-1: none) and its squared distance
  // (+inf: none), among the rows whose scan is < scan_below (INT64_MAX: all)
  void nearest(const double* queries, int64_t n, double max_distance, int64_t scan_below, int64_t* row, double* d2) {
    check(int(std::min<int64_t>(0, madicp_map_nearest(m_, queries, n, max_distance, scan_below, row, d2))),
          "madicp_map_nearest");
  }
  // the same in device memory of the context's device (queries row-strided, float32 or float64), ready on
  // consumer_stream with no host sync
  void nearestDev(const void* queries, int64_t n, int64_t stride, bool is_f32, double max_distance, int64_t scan_below,
                  int64_t* row, double* d2, void* consumer_stream) {
    check(int(std::min<int64_t>(0, madicp_map_nearest_dev(m_, queries, n, stride, is_f32 ? 1 : 0, max_distance,
                                                           scan_below, row, d2, consumer_stream))),
          "madicp_map_nearest_dev");
  }

 private:
  madicp_map_t* m_ = nullptr;
};

// reference: class MADicp (odometry/mad_icp.h:41-79).  `update(tree)` under the reference's OpenMP loop
// becomes "make this keyframe resident and part of the next round" (thread-safe); `updateState()` runs the round
// on the device (search + linearise + reduce + solve).  `compute(iters)` is the whole loop in one launch.
class MADicp {
 public:
  MADicp(double min_ball, double rho_ker, double b_ratio, int num_threads, int device = 0, int max_keyframes = 16)
      : max_keyframes_(max_keyframes) {
    (void) num_threads;  // CPU thread count of the reference; parallelism here is the GPU grid
    check(madicp_create(&ctx_, device, max_keyframes), "madicp_create");
    check(madicp_set_params(ctx_, min_ball, rho_ker, b_ratio), "madicp_set_params");
    X_ = Matrix4d::Identity();
    resident_.assign(size_t(max_keyframes), {nullptr, 0});
    resetAdders();
  }
  ~MADicp() { madicp_destroy(ctx_); }
  MADicp(const MADicp&) = delete;
  MADicp& operator=(const MADicp&) = delete;

  void resetAdders() {  // mad_icp.cpp:41-49; also starts a new round: no keyframe enqueued yet
    std::memset(H_adder_, 0, sizeof(H_adder_));
    std::memset(b_adder_, 0, sizeof(b_adder_));
    std::lock_guard<std::mutex> lk(mu_);
    round_.clear();
  }
  // mad_icp.cpp:51-53: the moving leaves are the leaves of the current scan's tree
  void setMoving(const MADtree& current) {
    if (current.deviceHandle()) {
      if (current.deviceContext() != ctx_) throw Error("MADicp.setMoving: the tree lives on another context");
      check(madicp_set_moving_tree(ctx_, current.deviceHandle()), "madicp_set_moving_tree");
    } else {
      const ContainerType moving = current.leafMeans();
      check(madicp_set_moving(ctx_, moving[0].data(), int(moving.size())), "madicp_set_moving");
    }
    matched_.assign(size_t(current.numLeaves()), 0);
  }
  void init(const Matrix4d& moving_in_fixed = Matrix4d::Identity()) { X_ = moving_in_fixed; }  // :55-57
  // mad_icp.cpp:74-103: the reference calls this from several OpenMP threads at once (pipeline.cpp:180-183)
  void update(const MADtree* fixed_tree) {
    std::lock_guard<std::mutex> lk(mu_);
    round_.push_back(fixed_tree);
  }
  // mad_icp.cpp:105-117 (plus the linearisation of the enqueued keyframes)
  void updateState() {
    std::vector<const MADtree*> round;
    {
      std::lock_guard<std::mutex> lk(mu_);
      round = round_;
    }
    std::sort(round.begin(), round.end(), [](const MADtree* a, const MADtree* b) { return a->version() < b->version(); });
    syncSlots(round);
    double X[12];
    pose12(X_, X);
    check(madicp_linearize(ctx_, X, H_adder_, b_adder_, matched_.data()), "madicp_linearize");
    check(madicp_solve_update(ctx_, H_adder_, b_adder_, X), "madicp_solve_update");
    X_ = from12(X);
  }
  // The loop of Pipeline::compute / MADicpWrapper::compute (pipeline.cpp:166-193) in one launch.  `partial`: the
  // realtime budget cut the loop short, so the matched flags were never cleared (pipeline.cpp:167-176).
  // iters == 0 leaves X_ as init() set it (the reference's loop with no rounds).
  int compute(const std::vector<const MADtree*>& keyframes, int iters, bool partial = false) {
    if (iters <= 0) {
      std::fill(matched_.begin(), matched_.end(), uint8_t(0));
      std::memset(H_adder_, 0, sizeof(H_adder_));
      std::memset(b_adder_, 0, sizeof(b_adder_));
      weight_ = 1.0 / 0.0;
      return 0;
    }
    syncSlots(keyframes);
    double X[12];
    pose12(X_, X);
    int n = 0;
    if (iters > MADICP_MAX_ITERS) {  // more than one launch holds: the blocking call chains launches
      check(madicp_register(ctx_, iters, X, H_adder_, b_adder_, matched_.data(), &n), "madicp_register");
      weight_ = 0.0;
    } else {
      check(partial ? madicp_register_partial_async(ctx_, iters, X) : madicp_register_async(ctx_, iters, X), "madicp_register");
      check(madicp_register_fetch_weight(ctx_, X, H_adder_, b_adder_, matched_.data(), &n, &weight_), "madicp_register_fetch");
    }
    X_ = from12(X);
    return n;
  }
  const std::vector<uint8_t>& matched() const { return matched_; }
  // Frame::weight_ = det(H_adder_^-1) of the last compute() (pipeline.cpp:223), from the device's solve thread
  double weight() const { return weight_; }
  madicp_ctx_t* context() { return ctx_; }

  Matrix4d X_;          // reference: Eigen::Isometry3d X_
  double H_adder_[36];  // reference: Matrix6d H_adder_ (H[r*6+c])
  double b_adder_[6];

 private:
  // keep exactly `trees` resident (a tree already in a slot with the same version is not re-uploaded); uploads
  // are asynchronous and apply the tree's pose on the device
  void syncSlots(const std::vector<const MADtree*>& trees) {
    if (int(trees.size()) > max_keyframes_) throw Error("more keyframes than slots");
    std::vector<char> keep(resident_.size(), 0);
    std::vector<const MADtree*> todo;
    for (const MADtree* t : trees) {
      bool found = false;
      for (size_t s = 0; s < resident_.size(); ++s)
        if (resident_[s].first && resident_[s].second == t->version() && !keep[s]) {
          keep[s] = 1;
          found = true;
          break;
        }
      if (!found) todo.push_back(t);
    }
    for (size_t s = 0; s < resident_.size(); ++s)
      if (!keep[s] && resident_[s].first) {
        check(madicp_drop_keyframe(ctx_, int(s)), "madicp_drop_keyframe");
        resident_[s] = {nullptr, 0};
      }
    for (const MADtree* t : todo)
      for (size_t s = 0; s < resident_.size(); ++s)
        if (!resident_[s].first) {
          if (t->deviceHandle())
            check(madicp_put_keyframe_tree(ctx_, int(s), t->deviceHandle(), t->pose()), "madicp_put_keyframe_tree");
          else
            check(madicp_put_keyframe_transformed(ctx_, int(s), t->hostHandle(), t->pose()), "madicp_put_keyframe");
          resident_[s] = {t, t->version()};
          break;
        }
  }
  madicp_ctx_t* ctx_ = nullptr;
  int max_keyframes_;
  std::vector<uint8_t> matched_;
  std::mutex mu_;
  std::vector<const MADtree*> round_;
  std::vector<std::pair<const MADtree*, uint64_t>> resident_;
  double weight_ = 0.0;
};

// reference: pybind/tools/mad_icp_wrapper.h:33-112
class MADicpWrapper {
 public:
  explicit MADicpWrapper(int num_threads, int device = 0) : num_threads_(num_threads), device_(device) {}
  void setQueryCloud(const ContainerType& query, double b_max, double b_min) {  // :40-45
    query_tree_.reset(new MADtree(query, b_max, b_min, levels()));  // (the reference never clears query_leaves_; here
  }                                                          //  a new cloud replaces the old one)
  void setReferenceCloud(const ContainerType& reference, double b_max, double b_min) {  // :47-52
    ref_b_max_ = b_max;
    ref_tree_.reset(new MADtree(reference, b_max, b_min, levels()));
  }
  Matrix4d compute(const Matrix4d& T, size_t max_icp_iterations, double rho_ker, double b_ratio, bool print_stats) {
    if (!ref_tree_ || !query_tree_) throw Error("MADicp.compute: set the reference and the query cloud first");
    if (!icp_ || rho_ker != rho_ker_ || b_ratio != b_ratio_ || ref_b_max_ != icp_b_max_) {
      icp_.reset(new MADicp(ref_b_max_, rho_ker, b_ratio, 1, device_, 1));  // :59
      rho_ker_ = rho_ker;
      b_ratio_ = b_ratio;
      icp_b_max_ = ref_b_max_;
    }
    icp_->setMoving(*query_tree_);
    icp_->init(T);
    const int matched = icp_->compute({ref_tree_.get()}, int(max_icp_iterations));  // :72-81
    if (print_stats) {                                                               // :87-99
      const int n = query_tree_->numLeaves();
      std::printf("MADicp|inliers ratio %g\n--MADicp|matched leaves %d\n--MADicp|total num leaves %d\n",
                  double(matched) / double(n), matched, n);
    }
    return icp_->X_;
  }

 private:
  int levels() const {  // max_parallel_levels_ = log2(num_threads) (mad_icp_wrapper.h:36)
    int l = 0;
    while ((2 << l) <= num_threads_) ++l;
    return l;
  }
  std::unique_ptr<MADicp> icp_;
  std::unique_ptr<MADtree> ref_tree_, query_tree_;
  double ref_b_max_ = 0.2, icp_b_max_ = -1, rho_ker_ = -1, b_ratio_ = -1;
  int num_threads_, device_;
};

// reference: pybind/tools/mad_tree_wrapper.h:34-71
class MADtreeWrapper {
 public:
  explicit MADtreeWrapper(int device = 0) : device_(device) {}
  ~MADtreeWrapper() {
    if (ctx_) madicp_destroy(ctx_);
  }
  void build(const ContainerType& vec, double b_max, double b_min, int max_parallel_level) {
    tree_.reset(new MADtree(vec, b_max, b_min, max_parallel_level));
    if (!ctx_) check(madicp_create(&ctx_, device_, 1), "madicp_create");
    check(madicp_put_keyframe(ctx_, 0, tree_->hostHandle()), "madicp_put_keyframe");
  }
  struct Matches {
    ContainerType points, normals;
    std::vector<double> dists;
  };
  // searchCloud / searchCloudDist (:48-67): (leaf mean, leaf normal[, distance]) per query
  Matches searchCloud(const ContainerType& queries, bool want_dist) {
    if (!tree_) throw Error("MADtree.search: build the tree first");
    Matches m;
    m.points.resize(queries.size());
    m.normals.resize(queries.size());
    if (want_dist) m.dists.resize(queries.size());
    if (!queries.empty())
      check(madicp_search_cloud(ctx_, 0, queries[0].data(), int64_t(queries.size()), nullptr, m.points[0].data(),
                                m.normals[0].data(), want_dist ? m.dists.data() : nullptr), "madicp_search_cloud");
    return m;
  }
  // the same for n queries in device memory (x, y, z at q + i * stride bytes), written to device outputs, ready on `stream`
  void searchCloudDev(const void* q, int64_t n, int64_t stride, bool is_f32, double* points, double* normals, double* dists,
                      void* stream) {
    if (!tree_) throw Error("MADtree.search: build the tree first");
    if (n > 0)
      check(madicp_search_cloud_dev(ctx_, 0, q, n, stride, is_f32 ? 1 : 0, nullptr, points, normals, dists, stream),
            "madicp_search_cloud_dev");
  }

 private:
  std::unique_ptr<MADtree> tree_;
  madicp_ctx_t* ctx_ = nullptr;
  int device_;
};

}  // namespace madicp_b200
