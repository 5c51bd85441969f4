// =============================================================================
// oracle/ref_capi.cpp -- TEST INFRASTRUCTURE, NOT PRODUCT CODE.
//
// C entry points over the UNMODIFIED reference classes (MADtree, MADicp, Pipeline), whose sources
// are compiled where they lie in a checkout of the reference by oracle/Makefile (target _ref) against
// oracle/eigen_standin (no Eigen installation needed).  The entry points mirror the orc_* functions of
// oracle_capi.cpp one for one, so tests/test_reference_pin.py can run the reference and the
// restatement on the same inputs and compare them coefficient by coefficient.
//
// Only the driver loop of ref_icp_run is written here: the reference keeps it inside
// Pipeline::compute (pipeline.cpp:166-193) and in a pybind header; it is restated below with the
// reference's MADicp calls, OpenMP shape included.
// =============================================================================
#include <odometry/mad_icp.h>
#include <odometry/pipeline.h>
#include <tools/constants.h>

#include <chrono>
#include <deque>
#include <unordered_map>

namespace {
struct TreeHandle {
  ContainerType cloud;
  MADtree* root = nullptr;
  LeafList leaves;
  std::unordered_map<const MADtree*, int> ordinal;
  ~TreeHandle() { delete root; }
};
void preorder(const MADtree* n, std::vector<const MADtree*>& out) {
  out.push_back(n);
  if (n->left_) preorder(n->left_, out);
  if (n->right_) preorder(n->right_, out);
}
Eigen::Isometry3d iso_from_rowmajor12(const double* X) {
  Eigen::Isometry3d T;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T.linear()(r, c) = X[r * 4 + c];
    T.translation()(r) = X[r * 4 + 3];
  }
  return T;
}
void iso_to_rowmajor12(const Eigen::Isometry3d& T, double* X) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) X[r * 4 + c] = T.linear()(r, c);
    X[r * 4 + 3] = T.translation()(r);
  }
}
// Pipeline keeps its state protected; a derived type may read it.
struct PipelineProbe : Pipeline {
  using Pipeline::Pipeline;
  size_t numKeyframes() const { return keyframes_.size(); }
  const Vector6d& velocity() const { return current_velocity_; }
  const Eigen::Isometry3d& pose() const { return frame_to_map_; }
  void deskewCloud(ContainerType* c, const Eigen::Isometry3d& a, const Eigen::Isometry3d& b) { deskew(c, a, b); }
  // pipeline.cpp:197-204, over the flags the last compute left on current_leaves_ (NaN before the first registration)
  double inliersRatio() const {
    if (current_leaves_.empty()) return std::nan("");
    int matched_leaves = 0;
    for (MADtree* l : current_leaves_)
      if (l->matched_) matched_leaves++;
    return double(matched_leaves) / double(current_leaves_.size());
  }
  const std::deque<Frame*>& frames() const { return frames_; }
  const std::deque<Frame*>& keyframes() const { return keyframes_; }
};
}  // namespace

extern "C" {

void* ref_tree_build(const double* pts, int n, double b_max, double b_min, int max_parallel_level) {
  TreeHandle* h = new TreeHandle;
  h->cloud.resize(n);
  for (int i = 0; i < n; ++i) h->cloud[i] = Eigen::Vector3d(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
  h->root = new MADtree(&h->cloud, h->cloud.begin(), h->cloud.end(), b_max, b_min, 0, max_parallel_level, nullptr, nullptr);
  h->root->getLeafs(std::back_insert_iterator<LeafList>(h->leaves));
  for (size_t i = 0; i < h->leaves.size(); ++i) h->ordinal[h->leaves[i]] = int(i);
  return h;
}
void ref_tree_free(void* t) { delete static_cast<TreeHandle*>(t); }
int ref_tree_num_leaves(void* t) { return int(static_cast<TreeHandle*>(t)->leaves.size()); }
int ref_tree_num_nodes(void* t) {
  std::vector<const MADtree*> v;
  preorder(static_cast<TreeHandle*>(t)->root, v);
  return int(v.size());
}
void ref_tree_cloud(void* t, double* out) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  for (size_t i = 0; i < h->cloud.size(); ++i)
    for (int j = 0; j < 3; ++j) out[3 * i + j] = h->cloud[i](j);
}
void ref_tree_apply_transform(void* t, const double* X12) {
  const Eigen::Isometry3d T = iso_from_rowmajor12(X12);
  static_cast<TreeHandle*>(t)->root->applyTransform(T.linear(), T.translation());
}
// same layout as orc_tree_export: DFS pre-order, eigenvectors column-major
void ref_tree_export(void* t, double* mean, double* eivecs, double* bbox, int* num_points, int* left, int* right,
                     int* leaf_ordinal) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  std::vector<const MADtree*> v;
  preorder(h->root, v);
  std::unordered_map<const MADtree*, int> pos;
  for (size_t i = 0; i < v.size(); ++i) pos[v[i]] = int(i);
  for (size_t i = 0; i < v.size(); ++i) {
    const MADtree* n = v[i];
    for (int j = 0; j < 3; ++j) {
      mean[3 * i + j] = n->mean_(j);
      bbox[3 * i + j] = n->bbox_(j);
    }
    for (int c = 0; c < 3; ++c)
      for (int r = 0; r < 3; ++r) eivecs[9 * i + c * 3 + r] = n->eigenvectors_(r, c);
    num_points[i] = n->num_points_;
    left[i] = n->left_ ? pos[n->left_] : -1;
    right[i] = n->right_ ? pos[n->right_] : -1;
    auto it = h->ordinal.find(n);
    leaf_ordinal[i] = (it == h->ordinal.end()) ? -1 : it->second;
  }
}
void ref_tree_search(void* t, const double* q, int n, int* ordinal_out) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  for (int i = 0; i < n; ++i) {
    const Eigen::Vector3d p(q[3 * i], q[3 * i + 1], q[3 * i + 2]);
    ordinal_out[i] = h->ordinal[h->root->bestMatchingLeafFast(p)];
  }
}

// The reference's registration loop (pipeline.cpp:166-193; for K = 1 it is mad_icp_wrapper.h:72-81).
// Outputs as orc_icp_run: X_hist = pose before each iteration, H/b after updateState (H column-major).
double ref_icp_run(void** keyframes, int K, void* moving, const double* X0, int iters, double min_ball, double rho_ker,
                   double b_ratio, int num_threads, double* X_final, double* X_hist, double* H_hist, double* b_hist,
                   unsigned char* matched, int* idx_hist) {
  std::deque<Frame*> frames;
  for (int k = 0; k < K; ++k) {
    Frame* f = new Frame;
    f->tree_ = static_cast<TreeHandle*>(keyframes[k])->root;
    frames.push_back(f);
  }
  TreeHandle* mv = static_cast<TreeHandle*>(moving);
  for (MADtree* l : mv->leaves) l->matched_ = false;
  omp_set_num_threads(num_threads);
  MADicp icp(min_ball, rho_ker, b_ratio, num_threads);
  icp.setMoving(mv->leaves);
  icp.init(iso_from_rowmajor12(X0));
  double seconds = 0.0;
  for (int it = 0; it < iters; ++it) {
    if (X_hist) iso_to_rowmajor12(icp.X_, X_hist + 12 * it);
    if (idx_hist) {  // the reference's OWN correspondences of this round (mad_icp.cpp:78-79), as getLeafs ordinals;
                     // outside the timed region
      const size_t L = mv->leaves.size();
      for (int k = 0; k < K; ++k) {
        TreeHandle* kf = static_cast<TreeHandle*>(keyframes[k]);
#pragma omp parallel for
        for (size_t q = 0; q < L; ++q) {
          const Eigen::Vector3d moving_leaf = icp.X_ * mv->leaves[q]->mean_;
          idx_hist[(size_t(it) * K + k) * L + q] = kf->ordinal.find(kf->root->bestMatchingLeafFast(moving_leaf))->second;
        }
      }
    }
    const auto t0 = std::chrono::steady_clock::now();
    if (it == iters - 1)
      for (MADtree* l : mv->leaves) l->matched_ = false;
    icp.resetAdders();
#pragma omp parallel for
    for (const Frame* frame : frames) {
      icp.update(frame->tree_);
    }
    icp.updateState();
    seconds += std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
    if (H_hist) std::memcpy(H_hist + 36 * it, icp.H_adder_.data(), sizeof(double) * 36);
    if (b_hist) std::memcpy(b_hist + 6 * it, icp.b_adder_.data(), sizeof(double) * 6);
  }
  iso_to_rowmajor12(icp.X_, X_final);
  if (matched)
    for (size_t q = 0; q < mv->leaves.size(); ++q) matched[q] = mv->leaves[q]->matched_ ? 1 : 0;
  for (Frame* f : frames) delete f;
  return seconds;
}

void* ref_pipeline_create(double sensor_hz, int deskew, double b_max, double rho_ker, double p_th, double b_min,
                          double b_ratio, int num_keyframes, int num_threads, int realtime) {
  return new PipelineProbe(sensor_hz, deskew != 0, b_max, rho_ker, p_th, b_min, b_ratio, num_keyframes, num_threads,
                           realtime != 0);
}
void ref_pipeline_free(void* p) { delete static_cast<PipelineProbe*>(p); }
void ref_pipeline_compute(void* p, double stamp, const double* pts, int n) {
  ContainerType cloud(n);
  for (int i = 0; i < n; ++i) cloud[i] = Eigen::Vector3d(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
  static_cast<PipelineProbe*>(p)->compute(stamp, cloud);
}
// as orc_pipeline_state; out[16] (inliers ratio, a local of Pipeline::compute) is recounted from the leaves' flags
void ref_pipeline_state(void* p, double* out) {
  PipelineProbe* P = static_cast<PipelineProbe*>(p);
  iso_to_rowmajor12(P->pose(), out);
  out[12] = P->isMapUpdated() ? 1 : 0;
  out[13] = double(P->currentID());
  out[14] = double(P->keyframeID());
  out[15] = double(P->numKeyframes());
  out[16] = P->inliersRatio();
  for (int i = 0; i < 6; ++i) out[17 + i] = P->velocity()(i);
}
// The frames window (frames_, oldest first): each frame's frame_ id and weight_ (either nullable); returns its size.
int ref_pipeline_frames(void* p, int* ids, double* weights) {
  const std::deque<Frame*>& f = static_cast<PipelineProbe*>(p)->frames();
  for (size_t i = 0; i < f.size(); ++i) {
    if (ids) ids[i] = f[i]->frame_;
    if (weights) weights[i] = f[i]->weight_;
  }
  return int(f.size());
}
// keyframes_ in their order: each keyframe's frame_ id (nullable); returns their number
int ref_pipeline_keyframes(void* p, int* ids) {
  const std::deque<Frame*>& f = static_cast<PipelineProbe*>(p)->keyframes();
  if (ids)
    for (size_t i = 0; i < f.size(); ++i) ids[i] = f[i]->frame_;
  return int(f.size());
}
// currentLeaves() (model == 0) or modelLeaves() as N x 3 doubles (out nullable); returns N
int ref_pipeline_leaves(void* p, int model, double* out) {
  PipelineProbe* P = static_cast<PipelineProbe*>(p);
  const ContainerType l = model ? P->modelLeaves() : P->currentLeaves();
  if (out)
    for (size_t i = 0; i < l.size(); ++i)
      for (int j = 0; j < 3; ++j) out[3 * i + j] = l[i](j);
  return int(l.size());
}
// trajectory(): every pose as 3 x 4 row-major (out nullable); returns their number
int ref_pipeline_trajectory(void* p, double* out) {
  const std::vector<Eigen::Isometry3d>& t = static_cast<PipelineProbe*>(p)->trajectory();
  if (out)
    for (size_t i = 0; i < t.size(); ++i) iso_to_rowmajor12(t[i], out + 12 * i);
  return int(t.size());
}
void ref_pipeline_deskew(void* p, double* pts, int n, const double* Tprev12, const double* Tnow12) {
  ContainerType c(n);
  for (int i = 0; i < n; ++i) c[i] = Eigen::Vector3d(pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]);
  static_cast<PipelineProbe*>(p)->deskewCloud(&c, iso_from_rowmajor12(Tprev12), iso_from_rowmajor12(Tnow12));
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts[3 * i + j] = c[i](j);
}
int ref_max_threads() { return omp_get_max_threads(); }

// The keyframe weight of pipeline.cpp:223, H_adder_.inverse().determinant(), for a row-major H.
double ref_inverse_determinant(const double* H36) {
  Eigen::Matrix<double, 6, 6> H;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) H(r, c) = H36[r * 6 + c];
  return H.inverse().determinant();
}

}  // extern "C"
