// reference_backend.cpp -- the CUDA backend as a drop-in replacement for TWO translation units of
// rvp-group/mad-icp: tools/mad_tree.cpp and odometry/mad_icp.cpp.
//
// It is compiled against the reference's OWN, UNMODIFIED headers (<tools/mad_tree.h>, <odometry/mad_icp.h>) and
// defines every member function those two files define -- same class layouts, same public data (X_, H_adder_,
// b_adder_, moving_leaves_, the pointer-linked MADtree nodes with mean_/eigenvectors_/bbox_/matched_) -- so the
// reference's odometry/pipeline.cpp, vel_estimator.cpp, the pybind wrappers and bin_runner compile and link
// against it unchanged (INTEGRATION.md section 2; the `ref_gpu` target of the test Makefile does exactly that and
// tests/test_gpu_adapter.py streams scans through the result).  Works with Eigen or any stand-in that offers
// coefficient access (`v(i)`, `m(r,c)`, `iso.linear()`, `iso.translation()`, `setZero`, `setIdentity`).
//
// What runs where:
//   MADtree::MADtree/build    host flat-tree builder of libmadicp_b200.so (bit-identical tree), then the
//                             reference's pointer-linked nodes are materialised from it (Pipeline reads
//                             leaf->mean_, leaf->matched_ and deletes trees node by node, mad_tree.h:58-63)
//   MADtree::applyTransform   the reference's arithmetic on the host nodes (modelLeaves() reads them) + the pose is
//                             remembered: the GPU copy is transformed on the device at promotion
//   MADicp::update(tree)      called concurrently under `#pragma omp parallel for` (pipeline.cpp:180-183): records
//                             the keyframe under a mutex, nothing else
//   MADicp::updateState()     makes the recorded keyframes resident (uploads only trees not yet on the GPU), then
//                             ONE persistent-kernel launch = search + linearise + reduce + solve for this round;
//                             writes X_, H_adder_, b_adder_ and sets moving->matched_ like mad_icp.cpp:85
// Host-only state that the reference's class layout has no room for (GPU context, flat trees) lives in side
// tables keyed by object address.
#include <odometry/mad_icp.h>
#include <tools/constants.h>
#include <tools/mad_tree.h>

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "../../../include/madicp_b200.h"

static_assert(sizeof(Eigen::Vector3d) == 3 * sizeof(double), "clouds are read as contiguous N x 3 doubles");

namespace {

void check(int rc, const char* what) {
  if (rc < 0) throw std::runtime_error(std::string(what) + " failed (" + std::to_string(rc) + "): " + madicp_last_error());
}

// ---------------------------------------------------------------- side table: trees
struct TreeState {
  madtree_t* flat = nullptr;  // sensor-frame flat tree (what the GPU gets)
  uint64_t uid = 0;           // creation order; also tells a new tree at a recycled address from the old one
  bool has_pose = false;      // applyTransform was called: the GPU copy is transformed at upload
  double X[12];
};
std::mutex g_mu;
std::unordered_map<const MADtree*, TreeState> g_trees;
uint64_t g_next_uid = 1;

void pose12(const Eigen::Matrix3d& r, const Eigen::Vector3d& t, double X[12]) {
  for (int i = 0; i < 3; ++i) {
    for (int j = 0; j < 3; ++j) X[i * 4 + j] = r(i, j);
    X[i * 4 + 3] = t(i);
  }
}

// ---------------------------------------------------------------- side table: MADicp objects
struct IcpState {
  madicp_ctx_t* ctx = nullptr;
  std::vector<const MADtree*> round;                      // keyframes recorded by update() since resetAdders()
  std::vector<std::pair<const MADtree*, uint64_t>> slot;  // resident tree per GPU slot (null = free)
  std::vector<double> means;
  std::vector<uint8_t> matched;
  const MADtree* moving_first = nullptr;  // identity of the uploaded moving set
  size_t moving_n = 0;
  bool moving_dirty = true;
};
std::unordered_map<const MADicp*, IcpState> g_icps;
constexpr int kSlots = 64;

IcpState& icp_state(const MADicp* self) { return g_icps[self]; }

}  // namespace

// ======================================================================================= MADtree
// tools/mad_tree.cpp:33-45
MADtree::MADtree(const ContainerTypePtr vec, const IteratorType begin, const IteratorType end, const double b_max,
                 const double b_min, const int level, const int max_parallel_level, MADtree* parent,
                 MADtree* plane_predecessor) {
  build(vec, begin, end, b_max, b_min, level, max_parallel_level, parent, plane_predecessor);
}

// tools/mad_tree.cpp:47-130.  Only whole trees are built (level 0, no parent): that is the only way the
// reference's callers use the constructor (pipeline.cpp:140-141,272-273; mad_icp_wrapper.h:42,50;
// mad_tree_wrapper.h:41).  The caller's vector is read, not reordered.
void MADtree::build(const ContainerTypePtr, const IteratorType begin, const IteratorType end, const double b_max,
                    const double b_min, const int level, const int max_parallel_level, MADtree* parent, MADtree*) {
  if (level != 0 || parent) throw std::logic_error("MADtree (CUDA backend): only whole trees can be built");
  const int64_t n = int64_t(end - begin);
  madtree_t* flat = nullptr;
  check(madtree_build(n > 0 ? &(*begin)(0) : nullptr, n, b_max, b_min, 1 << std::max(0, max_parallel_level), &flat),
        "madtree_build");
  const int N = madtree_num_nodes(flat);
  std::vector<double> mean(3 * size_t(N)), ev(9 * size_t(N)), bbox(3 * size_t(N));
  const size_t un = size_t(N);
  std::vector<int32_t> npts(un), left(un), right(un), ordinal(un);
  check(madtree_export(flat, mean.data(), ev.data(), bbox.data(), npts.data(), left.data(), right.data(), ordinal.data()),
        "madtree_export");
  // pointer-linked nodes in DFS pre-order (node 0 = this); children are plain `new` because the reference's inline
  // destructor deletes them one by one
  std::vector<MADtree*> node(size_t(N), nullptr);
  node[0] = this;
  for (int i = 0; i < N; ++i) {
    MADtree* m = node[size_t(i)];
    m->num_points_ = npts[size_t(i)];
    m->matched_ = false;
    for (int a = 0; a < 3; ++a) {
      m->mean_(a) = mean[size_t(i) * 3 + a];
      m->bbox_(a) = bbox[size_t(i) * 3 + a];
      for (int c = 0; c < 3; ++c) m->eigenvectors_(a, c) = ev[size_t(i) * 9 + c * 3 + a];
    }
    m->left_ = m->right_ = nullptr;
    if (left[size_t(i)] >= 0) {
      m->left_ = node[size_t(left[size_t(i)])] = new MADtree();
      m->left_->parent_ = m;
      m->right_ = node[size_t(right[size_t(i)])] = new MADtree();
      m->right_->parent_ = m;
    }
  }
  parent_ = nullptr;
  std::lock_guard<std::mutex> lk(g_mu);
  TreeState& st = g_trees[this];
  if (st.flat) madtree_free(st.flat);  // a deleted tree's address, recycled by the allocator
  st = TreeState{};
  st.flat = flat;
  st.uid = g_next_uid++;
  // Trees die inside the reference's inline destructor, where no backend code runs.  Entries that are neither
  // among the FRAME_WINDOW + 2 newest nor resident on a GPU (checked by updateState) are certainly dead.
  if (g_trees.size() > size_t(FRAME_WINDOW + 2 + kSlots + 8)) {
    std::vector<std::pair<uint64_t, const MADtree*>> by_age;
    for (const auto& kv : g_trees) by_age.push_back({kv.second.uid, kv.first});
    std::sort(by_age.begin(), by_age.end());
    for (size_t i = 0; i + size_t(FRAME_WINDOW + 2 + kSlots) < by_age.size(); ++i) {
      bool resident = false;
      for (const auto& ic : g_icps)
        for (const auto& s : ic.second.slot) resident |= (s.first == by_age[i].second && s.second == by_age[i].first);
      if (resident) continue;
      madtree_free(g_trees[by_age[i].second].flat);
      g_trees.erase(by_age[i].second);
    }
  }
}

// tools/mad_tree.cpp:132-142
MADtree* MADtree::makeSubtree(const ContainerTypePtr vec, const IteratorType begin, const IteratorType end,
                              const double b_max, const double b_min, const int level, const int max_parallel_level,
                              MADtree* parent, MADtree* plane_predecessor) {
  return new MADtree(vec, begin, end, b_max, b_min, level, max_parallel_level, parent, plane_predecessor);
}

// tools/mad_tree.cpp:144-152 (host walk over the pointer-linked nodes; the GPU walk is madicp_search_cloud)
const MADtree* MADtree::bestMatchingLeafFast(const Eigen::Vector3d& query) const {
  const MADtree* at = this;
  for (;;) {
    if (!at->left_ && !at->right_) return at;
    double s = 0.0;  // (query - mean_) . eigenvectors_.col(2), summed as ((x + y) + z)
    s = (query(0) - at->mean_(0)) * at->eigenvectors_(0, 2) + (query(1) - at->mean_(1)) * at->eigenvectors_(1, 2);
    s = s + (query(2) - at->mean_(2)) * at->eigenvectors_(2, 2);
    at = (s < 0.0) ? at->left_ : at->right_;
  }
}

// tools/mad_tree.cpp:154-163
void MADtree::getLeafs(std::back_insert_iterator<std::vector<MADtree*>> it) {
  std::vector<MADtree*> stack{this};
  while (!stack.empty()) {
    MADtree* m = stack.back();
    stack.pop_back();
    if (!m->left_ && !m->right_) {
      ++it = m;
      continue;
    }
    if (m->right_) stack.push_back(m->right_);
    if (m->left_) stack.push_back(m->left_);  // left subtree first, as the reference's recursion
  }
}

// tools/mad_tree.cpp:165-172
void MADtree::applyTransform(const Eigen::Matrix3d& r, const Eigen::Vector3d& t) {
  std::vector<MADtree*> stack{this};
  while (!stack.empty()) {
    MADtree* m = stack.back();
    stack.pop_back();
    m->mean_ = r * m->mean_ + t;
    m->eigenvectors_ = r * m->eigenvectors_;
    if (m->left_) stack.push_back(m->left_);
    if (m->right_) stack.push_back(m->right_);
  }
  if (parent_) return;  // a subtree: no GPU-side identity
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_trees.find(this);
  if (it == g_trees.end()) return;
  TreeState& st = it->second;
  if (st.has_pose) check(madtree_apply_transform(st.flat, st.X), "madtree_apply_transform");  // (twice: not in Pipeline)
  pose12(r, t, st.X);
  st.has_pose = true;
  st.uid = g_next_uid++;  // new content: a resident copy of the old one must not be reused
}

// ======================================================================================= MADicp
// odometry/mad_icp.cpp:31-39
MADicp::MADicp(double min_ball, double rho_ker, double b_ratio, int num_threads)
  : rho_ker_(sqrt(rho_ker)), min_ball_(min_ball), b_ratio_(b_ratio), num_threads_(num_threads) {
  X_.setIdentity();
  H_adder_.setZero();
  b_adder_.setZero();
  H_adders_ = std::vector<Matrix6d>(size_t(num_threads));  // kept for layout compatibility; the GPU sums directly
  b_adders_ = std::vector<Vector6d>(size_t(num_threads));
  for (auto& h : H_adders_) h.setZero();
  for (auto& b : b_adders_) b.setZero();
  std::lock_guard<std::mutex> lk(g_mu);
  IcpState& st = icp_state(this);
  if (st.ctx) madicp_destroy(st.ctx);  // an earlier object at this address (MADicp has no user destructor to hook)
  st = IcpState{};
  const char* dev = std::getenv("MADICP_DEVICE");
  check(madicp_create(&st.ctx, dev ? std::atoi(dev) : 0, kSlots), "madicp_create");
  check(madicp_set_params(st.ctx, min_ball, rho_ker, b_ratio), "madicp_set_params");
  st.slot.assign(size_t(kSlots), {nullptr, 0});
}

// odometry/mad_icp.cpp:41-49
void MADicp::resetAdders() {
  H_adder_.setZero();
  b_adder_.setZero();
  std::lock_guard<std::mutex> lk(g_mu);
  icp_state(this).round.clear();
}

// odometry/mad_icp.cpp:51-53
void MADicp::setMoving(const LeafList& moving_leaves) {
  moving_leaves_ = moving_leaves;
  std::lock_guard<std::mutex> lk(g_mu);
  icp_state(this).moving_dirty = true;
}

// odometry/mad_icp.cpp:55-57
void MADicp::init(const Eigen::Isometry3d& moving_in_fixed) { X_ = moving_in_fixed; }

// odometry/mad_icp.cpp:59-72 (not used by the GPU path; kept because it is part of the class)
void MADicp::errorAndJacobian(double& e, JacobianMatrixType& J, const MADtree& fixed, const MADtree& moving,
                              const Eigen::Vector3d& moving_transformed) const {
  double n[3], d[3], Jt[3];
  for (int a = 0; a < 3; ++a) {
    n[a] = fixed.eigenvectors_(a, 0);
    d[a] = moving_transformed(a) - fixed.mean_(a);
  }
  e = (d[0] * n[0] + d[1] * n[1]) + d[2] * n[2];
  for (int c = 0; c < 3; ++c) {
    Jt[c] = (n[0] * X_.linear()(0, c) + n[1] * X_.linear()(1, c)) + n[2] * X_.linear()(2, c);
    J(0, c) = Jt[c];
  }
  const double px = moving.mean_(0), py = moving.mean_(1), pz = moving.mean_(2);
  J(0, 3) = -(Jt[1] * pz - Jt[2] * py);  // -J[0:3] * skew(p)
  J(0, 4) = -(Jt[2] * px - Jt[0] * pz);
  J(0, 5) = -(Jt[0] * py - Jt[1] * px);
}

// odometry/mad_icp.cpp:74-103 -- concurrent callers (one OpenMP thread per keyframe)
void MADicp::update(const MADtree* fixed_tree) {
  std::lock_guard<std::mutex> lk(g_mu);
  icp_state(this).round.push_back(fixed_tree);
}

// odometry/mad_icp.cpp:105-117 (+ the search / linearisation of the recorded keyframes)
void MADicp::updateState() {
  std::lock_guard<std::mutex> lk(g_mu);
  IcpState& st = icp_state(this);
  // moving leaves: uploaded once per setMoving()
  const size_t L = moving_leaves_.size();
  if (L == 0) throw std::logic_error("MADicp::updateState: no moving leaves");
  if (st.moving_dirty) {
    st.means.resize(L * 3);
    for (size_t i = 0; i < L; ++i)
      for (int a = 0; a < 3; ++a) st.means[i * 3 + size_t(a)] = moving_leaves_[i]->mean_(a);
    check(madicp_set_moving(st.ctx, st.means.data(), int(L)), "madicp_set_moving");
    st.matched.assign(L, 0);
    st.moving_dirty = false;
  }
  // keyframes of this round, in creation order (OpenMP gives no order; a fixed one keeps the sums reproducible)
  struct Want {
    const MADtree* t;
    uint64_t uid;
  };
  std::vector<Want> want;
  for (const MADtree* t : st.round) {
    auto it = g_trees.find(t);
    if (it == g_trees.end()) throw std::logic_error("MADicp::update: tree was not built by this backend");
    want.push_back({t, it->second.uid});
  }
  std::sort(want.begin(), want.end(), [](const Want& a, const Want& b) { return a.uid < b.uid; });
  if (want.size() > size_t(kSlots)) throw std::length_error("MADicp: more than 64 keyframes in one round");
  std::vector<char> keep(st.slot.size(), 0);
  std::vector<Want> todo;
  for (const Want& w : want) {
    bool found = false;
    for (size_t s = 0; s < st.slot.size() && !found; ++s)
      if (st.slot[s].first == w.t && st.slot[s].second == w.uid && !keep[s]) keep[s] = found = true;
    if (!found) todo.push_back(w);
  }
  for (size_t s = 0; s < st.slot.size(); ++s)
    if (!keep[s] && st.slot[s].first) {
      check(madicp_drop_keyframe(st.ctx, int(s)), "madicp_drop_keyframe");
      st.slot[s] = {nullptr, 0};
    }
  for (const Want& w : todo)
    for (size_t s = 0; s < st.slot.size(); ++s)
      if (!st.slot[s].first) {
        const TreeState& ts = g_trees[w.t];
        check(madicp_put_keyframe_transformed(st.ctx, int(s), ts.flat, ts.has_pose ? ts.X : nullptr), "madicp_put_keyframe");
        st.slot[s] = {w.t, w.uid};
        break;
      }
  // one round on the device
  double X[12], H[36], b[6];
  pose12(X_.linear(), X_.translation(), X);
  int n_matched = 0;
  check(madicp_register(st.ctx, 1, X, H, b, st.matched.data(), &n_matched), "madicp_register");
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) X_.linear()(r, c) = X[r * 4 + c];
    X_.translation()(r) = X[r * 4 + 3];
  }
  for (int r = 0; r < 6; ++r) {
    for (int c = 0; c < 6; ++c) H_adder_(r, c) = H[r * 6 + c];
    b_adder_(r) = b[r];
  }
  for (size_t i = 0; i < L; ++i)
    if (st.matched[i]) moving_leaves_[i]->matched_ = true;  // mad_icp.cpp:85 (sticky until Pipeline clears it)
}

// Optional clean-up hooks for hosts that want the GPU memory back before process exit (the reference's classes
// have no destructors this backend could use).
extern "C" void madicp_b200_backend_release_icp(const MADicp* icp) {
  std::lock_guard<std::mutex> lk(g_mu);
  auto it = g_icps.find(icp);
  if (it == g_icps.end()) return;
  if (it->second.ctx) madicp_destroy(it->second.ctx);
  g_icps.erase(it);
}
extern "C" void madicp_b200_backend_release_all() {
  std::lock_guard<std::mutex> lk(g_mu);
  for (auto& kv : g_icps)
    if (kv.second.ctx) madicp_destroy(kv.second.ctx);
  g_icps.clear();
  for (auto& kv : g_trees) madtree_free(kv.second.flat);
  g_trees.clear();
}
