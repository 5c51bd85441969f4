// =============================================================================
// oracle/oracle_capi.cpp -- TEST INFRASTRUCTURE (see madicp_oracle.hpp header).
// C entry points over the CPU restatement so tests/ and bench.py's cpu_baseline
// leg can drive it through ctypes.  Parity status: see madicp_oracle.hpp.
// =============================================================================
#include "madicp_oracle.hpp"

#include <chrono>
#include <unordered_map>

using namespace orc;

namespace {
struct TreeHandle {
  Cloud cloud;  // the (reordered, mutated) working copy the build wrote into
  Tree* root = nullptr;
  LeafList leaves;                                // DFS order (getLeafs)
  std::unordered_map<const Tree*, int> ordinal;  // leaf -> DFS ordinal
  ~TreeHandle() { delete root; }
};

void preorder(const Tree* n, std::vector<const Tree*>& out) {
  out.push_back(n);
  if (n->left_) preorder(n->left_, out);
  if (n->right_) preorder(n->right_, out);
}

Iso3 iso_from_rowmajor12(const double* X) {  // [R|t] 3x4 row-major
  Iso3 T;
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) T.R(r, c) = X[r * 4 + c];
    T.t[r] = X[r * 4 + 3];
  }
  return T;
}
void iso_to_rowmajor12(const Iso3& T, double* X) {
  for (int r = 0; r < 3; ++r) {
    for (int c = 0; c < 3; ++c) X[r * 4 + c] = T.R(r, c);
    X[r * 4 + 3] = T.t[r];
  }
}
}  // namespace

extern "C" {

// MADtree(vec, begin, end, b_max, b_min, 0, max_parallel_level, nullptr, nullptr)
void* orc_tree_build(const double* pts, int n, double b_max, double b_min) {
  TreeHandle* h = new TreeHandle;
  h->cloud.resize(n);
  for (int i = 0; i < n; ++i) h->cloud[i] = V3{{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]}};
  h->root = new Tree(&h->cloud, 0, size_t(n), b_max, b_min, 0, 0, nullptr, nullptr);
  h->root->getLeafs(h->leaves);
  for (size_t i = 0; i < h->leaves.size(); ++i) h->ordinal[h->leaves[i]] = int(i);
  return h;
}
void orc_tree_free(void* t) { delete static_cast<TreeHandle*>(t); }
int orc_tree_num_leaves(void* t) { return int(static_cast<TreeHandle*>(t)->leaves.size()); }
int orc_tree_num_nodes(void* t) {
  std::vector<const Tree*> v;
  preorder(static_cast<TreeHandle*>(t)->root, v);
  return int(v.size());
}
// cloud after the build's in-place reordering / leaf write (utils.h:47, mad_tree.cpp:82)
void orc_tree_cloud(void* t, double* out) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  for (size_t i = 0; i < h->cloud.size(); ++i)
    for (int j = 0; j < 3; ++j) out[3 * i + j] = h->cloud[i][j];
}
void orc_tree_apply_transform(void* t, const double* X12) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  const Iso3 T = iso_from_rowmajor12(X12);
  h->root->applyTransform(T.R, T.t);
}
// Leaves in getLeafs (DFS) order: mean, normal = eigenvectors.col(0), bbox(0), num_points
void orc_tree_leaves(void* t, double* means, double* normals, double* bbox0, int* num_points) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  for (size_t i = 0; i < h->leaves.size(); ++i) {
    const Tree* l = h->leaves[i];
    for (int j = 0; j < 3; ++j) {
      if (means) means[3 * i + j] = l->mean_[j];
      if (normals) normals[3 * i + j] = l->eigenvectors_(j, 0);
    }
    if (bbox0) bbox0[i] = l->bbox_[0];
    if (num_points) num_points[i] = l->num_points_;
  }
}
// All nodes in DFS pre-order: mean[3], eigenvectors[9] col-major, bbox[3], num_points,
// left/right pre-order index (-1 for leaves), leaf ordinal (-1 for internal nodes).
void orc_tree_export(void* t, double* mean, double* eivecs, double* bbox, int* num_points, int* left, int* right,
                     int* leaf_ordinal) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  std::vector<const Tree*> v;
  preorder(h->root, v);
  std::unordered_map<const Tree*, int> pos;
  for (size_t i = 0; i < v.size(); ++i) pos[v[i]] = int(i);
  for (size_t i = 0; i < v.size(); ++i) {
    const Tree* n = v[i];
    for (int j = 0; j < 3; ++j) {
      mean[3 * i + j] = n->mean_[j];
      bbox[3 * i + j] = n->bbox_[j];
    }
    for (int j = 0; j < 9; ++j) eivecs[9 * i + j] = n->eigenvectors_.m[j];
    num_points[i] = n->num_points_;
    left[i] = n->left_ ? pos[n->left_] : -1;
    right[i] = n->right_ ? pos[n->right_] : -1;
    auto it = h->ordinal.find(n);
    leaf_ordinal[i] = (it == h->ordinal.end()) ? -1 : it->second;
  }
}
// bestMatchingLeafFast for a batch; writes the DFS leaf ordinal and (nullable) the
// number of internal nodes visited (the d(q,k) of SURVEY 8d).
void orc_tree_search(void* t, const double* q, int n, int* ordinal_out, int* depth_out) {
  TreeHandle* h = static_cast<TreeHandle*>(t);
  for (int i = 0; i < n; ++i) {
    const V3 p{{q[3 * i], q[3 * i + 1], q[3 * i + 2]}};
    const Tree* leaf = h->root->bestMatchingLeafFast(p);
    ordinal_out[i] = h->ordinal[leaf];
    if (depth_out) {
      int d = 0;
      for (const Tree* n2 = leaf; n2->parent_; n2 = n2->parent_) ++d;
      depth_out[i] = d;
    }
  }
}

// -----------------------------------------------------------------------------
// Registration.  keyframes: K tree handles (fixed); moving: tree handle whose
// leaves are the moving leaves (query tree, sensor frame).  X0: 3x4 row-major.
// Outputs (all nullable except X_final):
//   X_hist   iters x 12   pose BEFORE each iteration (teacher forcing)
//   H_hist   iters x 36   H_adder_ (col-major) after each iteration's updateState
//   b_hist   iters x 6
//   idx_hist iters x K x L  DFS ordinal of bestMatchingLeafFast (before the gate)
//   matched  L            matched_ flags after the loop
// Returns seconds spent in the loop (recording off => this is the timed baseline).
// -----------------------------------------------------------------------------
double orc_icp_run(void** keyframes, int K, void* moving, const double* X0, int iters, double min_ball, double rho_ker,
                   double b_ratio, int num_threads, double* X_final, double* X_hist, double* H_hist, double* b_hist,
                   int* idx_hist, unsigned char* matched) {
  std::vector<Tree*> kfs(K);
  std::vector<TreeHandle*> kh(K);
  for (int k = 0; k < K; ++k) {
    kh[k] = static_cast<TreeHandle*>(keyframes[k]);
    kfs[k] = kh[k]->root;
  }
  TreeHandle* mv = static_cast<TreeHandle*>(moving);
  const size_t L = mv->leaves.size();
  for (Tree* l : mv->leaves) l->matched_ = false;
  MADicp icp(min_ball, rho_ker, b_ratio, num_threads);
  icp.setMoving(mv->leaves);
  icp.init(iso_from_rowmajor12(X0));
  const bool want_rec = X_hist || H_hist || b_hist || idx_hist;
  IcpRecord rec;
  const auto t0 = std::chrono::steady_clock::now();
  icp_loop(icp, kfs, mv->leaves, iters, num_threads, want_rec ? &rec : nullptr, idx_hist != nullptr);
  const auto t1 = std::chrono::steady_clock::now();
  iso_to_rowmajor12(icp.X_, X_final);
  for (int it = 0; it < iters && want_rec; ++it) {
    if (X_hist) iso_to_rowmajor12(rec.X_before[it], X_hist + 12 * it);
    if (H_hist) std::memcpy(H_hist + 36 * it, rec.H[it].m, sizeof(double) * 36);
    if (b_hist) std::memcpy(b_hist + 6 * it, rec.b[it].v, sizeof(double) * 6);
    if (idx_hist)
      for (int k = 0; k < K; ++k)
        for (size_t q = 0; q < L; ++q)
          idx_hist[(size_t(it) * K + k) * L + q] = kh[k]->ordinal[rec.matches[it][size_t(k) * L + q]];
  }
  if (matched)
    for (size_t q = 0; q < L; ++q) matched[q] = mv->leaves[q]->matched_ ? 1 : 0;
  return std::chrono::duration<double>(t1 - t0).count();
}

// One linearisation at a given pose (resetAdders + update over K keyframes, no
// updateState): returns the summed H (col-major 36), b (6) and matched flags.
void orc_icp_linearize(void** keyframes, int K, void* moving, const double* X, double min_ball, double rho_ker,
                       double b_ratio, double* H, double* b, unsigned char* matched) {
  TreeHandle* mv = static_cast<TreeHandle*>(moving);
  for (Tree* l : mv->leaves) l->matched_ = false;
  MADicp icp(min_ball, rho_ker, b_ratio, 1);
  icp.setMoving(mv->leaves);
  icp.init(iso_from_rowmajor12(X));
  icp.resetAdders();
  omp_set_num_threads(1);
  for (int k = 0; k < K; ++k) icp.update(static_cast<TreeHandle*>(keyframes[k])->root);
  std::memcpy(H, icp.H_adders_[0].m, sizeof(double) * 36);
  std::memcpy(b, icp.b_adders_[0].v, sizeof(double) * 6);
  if (matched)
    for (size_t q = 0; q < mv->leaves.size(); ++q) matched[q] = mv->leaves[q]->matched_ ? 1 : 0;
}

// H.ldlt().solve(-b), expMapSO3, X*dX  (mad_icp.cpp:111-116) exposed for unit tests
void orc_solve_update(const double* H36, const double* b6, const double* X12, double* dx6, double* Xout12) {
  M6 H;
  V6 nb, dx;
  std::memcpy(H.m, H36, sizeof(H.m));
  for (int i = 0; i < 6; ++i) nb.v[i] = -b6[i];
  ldlt6_solve(H, nb, dx);
  Iso3 dX;
  dX.R = expMapSO3(V3{{dx.v[3], dx.v[4], dx.v[5]}});
  dX.t = V3{{dx.v[0], dx.v[1], dx.v[2]}};
  const Iso3 Xn = isoMul(iso_from_rowmajor12(X12), dX);
  if (dx6) std::memcpy(dx6, dx.v, sizeof(double) * 6);
  iso_to_rowmajor12(Xn, Xout12);
}
void orc_eig3(const double* cov9_colmajor, double* eivecs9_colmajor, double* eivals3) {
  M3 c, e;
  std::memcpy(c.m, cov9_colmajor, sizeof(c.m));
  eig3_computeDirect(c, e, eivals3);
  std::memcpy(eivecs9_colmajor, e.m, sizeof(e.m));
}
void orc_expmap(const double* w3, double* R9_rowmajor) {
  const M3 R = expMapSO3(V3{{w3[0], w3[1], w3[2]}});
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) R9_rowmajor[r * 3 + c] = R(r, c);
}
int orc_max_threads() { return omp_get_max_threads(); }

}  // extern "C"

// -----------------------------------------------------------------------------
// Pipeline (the caller of the hot path): odometry/pipeline.{h,cpp}
// -----------------------------------------------------------------------------
#include "pipeline_oracle.hpp"
extern "C" {
void* orc_pipeline_create(double sensor_hz, int deskew, double b_max, double rho_ker, double p_th, double b_min,
                          double b_ratio, int num_keyframes, int num_threads, int realtime) {
  return new orc::Pipeline(sensor_hz, deskew != 0, b_max, rho_ker, p_th, b_min, b_ratio, num_keyframes, num_threads,
                           realtime != 0);
}
void orc_pipeline_free(void* p) { delete static_cast<orc::Pipeline*>(p); }
void orc_pipeline_compute(void* p, double stamp, const double* pts, int n) {
  static_cast<orc::Pipeline*>(p)->compute(stamp, pts, n);
}
// out: pose 3x4 row-major (12), then [is_map_updated, current_id, keyframe_id, num_keyframes, inliers_ratio,
// velocity(6)] (11 doubles)
void orc_pipeline_state(void* p, double* out) {
  orc::Pipeline* P = static_cast<orc::Pipeline*>(p);
  iso_to_rowmajor12(P->frame_to_map_, out);
  out[12] = P->is_map_updated_ ? 1 : 0;
  out[13] = double(P->seq_);
  out[14] = double(P->seq_keyframe_);
  out[15] = double(P->keyframes_.size());
  out[16] = P->last_inliers_ratio_;
  for (int i = 0; i < 6; ++i) out[17 + i] = P->current_velocity_.v[i];
}
}
// the keyframe weight (pipeline.cpp:223) of a row-major H, as the restated Pipeline computes it
extern "C" double orc_inverse_determinant6(const double* H36) {
  orc::M6 H;
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) H(r, c) = H36[r * 6 + c];
  return orc::inverseDeterminant6(H);
}
extern "C" void orc_pipeline_deskew(void* p, double* pts, int n, const double* Tprev12, const double* Tnow12) {
  orc::Cloud c(n);
  for (int i = 0; i < n; ++i) c[i] = V3{{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]}};
  static_cast<orc::Pipeline*>(p)->deskew(&c, iso_from_rowmajor12(Tprev12), iso_from_rowmajor12(Tnow12));
  for (int i = 0; i < n; ++i)
    for (int j = 0; j < 3; ++j) pts[3 * i + j] = c[i][j];
}
