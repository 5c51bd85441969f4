// =============================================================================
// oracle/pipeline_oracle.hpp -- TEST INFRASTRUCTURE (see madicp_oracle.hpp header).
// Eigen-free restatement of the reference's per-scan driver, the CALLER of the hot path:
//   odometry/pipeline.{h,cpp}  (initialize, deskew, compute: prediction, ICP loop, inlier ratio,
//                               velocity smoothing, keyframe selection by det(H^-1))
//   odometry/vel_estimator.{h,cpp}
//   tools/lie_algebra.h:54-89  logMapSO3
// Pinned bit for bit to the reference's sources built against oracle/eigen_standin
// (tests/test_reference_pin.py); Eigen's internal evaluation order stays unpinned (madicp_oracle.hpp).
// =============================================================================
#pragma once
#include <algorithm>
#include <deque>

#include "madicp_oracle.hpp"

namespace orc {

static constexpr int CHUNKS = 1024;              // tools/constants.h:31-35
static constexpr int SMOOTHING_T = 10;
static constexpr double E_THRESHOLD_VEL = 0.3162;
static constexpr int MAX_ICP_ITS = 15;
static constexpr int FRAME_WINDOW = 10;

inline Iso3 isoIdentity() {
  Iso3 I;
  I.R = identity3();
  I.t = V3{{0, 0, 0}};
  return I;
}
inline Iso3 isoInverse(const Iso3& T) {  // Isometry: R^T, -R^T t
  Iso3 I;
  for (int r = 0; r < 3; ++r)
    for (int c = 0; c < 3; ++c) I.R(r, c) = T.R(c, r);
  const V3 rt = mulMV(I.R, T.t);
  I.t = V3{{-rt[0], -rt[1], -rt[2]}};
  return I;
}
// tools/lie_algebra.h:54-89
inline V3 logMapSO3(const M3& R) {
  const double R11 = R(0, 0), R12 = R(0, 1), R13 = R(0, 2);
  const double R21 = R(1, 0), R22 = R(1, 1), R23 = R(1, 2);
  const double R31 = R(2, 0), R32 = R(2, 1), R33 = R(2, 2);
  const double tr = R11 + R22 + R33;
  const double pi(M_PI), two(2);
  V3 omega;
  if (tr + 1.0 < 1e-10) {
    double f;
    if (std::fabs(R33 + 1.0) > 1e-5) {
      f = pi / std::sqrt(two + two * R33);
      omega = V3{{f * R13, f * R23, f * (1.0 + R33)}};
    } else if (std::fabs(R22 + 1.0) > 1e-5) {
      f = pi / std::sqrt(two + two * R22);
      omega = V3{{f * R12, f * (1.0 + R22), f * R32}};
    } else {
      f = pi / std::sqrt(two + two * R11);
      omega = V3{{f * (1.0 + R11), f * R21, f * R31}};
    }
  } else {
    double magnitude;
    const double tr_3 = tr - 3.0;
    if (tr_3 < -1e-7) {
      const double theta = std::acos((tr - 1.0) / two);
      magnitude = theta / (two * std::sin(theta));
    } else {
      magnitude = 0.5 - tr_3 * tr_3 / 12.0;
    }
    omega = V3{{magnitude * (R32 - R23), magnitude * (R13 - R31), magnitude * (R21 - R12)}};
  }
  return omega;
}
// det(H^-1) via partial-pivot LU of H (pipeline.cpp:223 computes H.inverse().determinant())
inline double inverseDeterminant6(const M6& H) {
  double A[6][6];
  for (int r = 0; r < 6; ++r)
    for (int c = 0; c < 6; ++c) A[r][c] = H(r, c);
  double det = 1.0;
  for (int k = 0; k < 6; ++k) {
    int p = k;
    for (int i = k + 1; i < 6; ++i)
      if (std::fabs(A[i][k]) > std::fabs(A[p][k])) p = i;
    if (p != k) {
      for (int c = 0; c < 6; ++c) std::swap(A[k][c], A[p][c]);
      det = -det;
    }
    det *= A[k][k];
    for (int i = k + 1; i < 6; ++i) {
      const double f = A[i][k] / A[k][k];
      for (int c = k; c < 6; ++c) A[i][c] -= f * A[k][c];
    }
  }
  // a zero last pivot: the reference's inverse() divides by it and the determinant of that is NaN (not 1/+-0)
  return (A[5][5] == 0.0) ? std::numeric_limits<double>::quiet_NaN() : 1.0 / det;
}

// odometry/vel_estimator.{h,cpp}
struct VelEstimator {
  M6 H_adder_;
  V6 X_, b_adder_;
  std::vector<Iso3> odometry_;
  double ts_;
  explicit VelEstimator(double sensor_hz) : ts_(1. / sensor_hz) { std::memset(&X_, 0, sizeof(X_)); }
  void init(const V6& v) { X_ = v; }
  void setOdometry(const std::vector<Iso3>& o) { odometry_ = o; }
  void update(const Iso3& T_now, const Iso3& T_prev, double delta_t, double weight) {  // :63-79
    const Iso3 T = isoMul(isoInverse(T_prev), T_now);
    double e[6];
    for (int i = 0; i < 3; ++i) e[i] = delta_t * X_.v[i] - T.t[i];
    const double a0 = std::atan2(-T.R(1, 2), T.R(2, 2)), a1 = std::asin(T.R(0, 2)), a2 = std::atan2(-T.R(0, 1), T.R(0, 0));
    e[3] = delta_t * X_.v[3] - a0;
    e[4] = delta_t * X_.v[4] - a1;
    e[5] = delta_t * X_.v[5] - a2;
    double scale = 1.;
    double chi2 = 0;
    for (int i = 0; i < 6; ++i) chi2 += e[i] * e[i];
    const double chi = std::sqrt(chi2);
    if (chi > E_THRESHOLD_VEL) scale = E_THRESHOLD_VEL / chi;
    const double sw = scale * weight;
    for (int i = 0; i < 6; ++i) {  // J = I * delta_t
      H_adder_(i, i) += (sw * delta_t) * delta_t;
      b_adder_.v[i] += (sw * delta_t) * e[i];
    }
  }
  void oneRound() {  // :81-97
    std::memset(&H_adder_, 0, sizeof(H_adder_));
    std::memset(&b_adder_, 0, sizeof(b_adder_));
    const Iso3 T_now = odometry_.back();
    for (size_t i = 0; i + 1 < odometry_.size(); ++i) {
      const double delta_t = (odometry_.size() - 1 - i) * ts_;
      const double weight = 1.f - double(odometry_.size() - 2 - i) / double(odometry_.size() - 1);
      update(T_now, odometry_[i], delta_t, weight);
    }
    V6 nb, dx;
    for (int i = 0; i < 6; ++i) nb.v[i] = -b_adder_.v[i];
    ldlt6_solve(H_adder_, nb, dx);
    for (int i = 0; i < 6; ++i) X_.v[i] += dx.v[i];
  }
};

struct Frame {  // tools/frame.h:37-51
  Iso3 frame_to_map_ = isoIdentity();
  Tree* tree_ = nullptr;
  LeafList leaves_;
  Cloud* cloud_ = nullptr;  // storage the tree was built over (kept alive with the tree)
  double stamp_ = 0., weight_ = 0.;
  int frame_ = 0;
};

// odometry/pipeline.{h,cpp}
struct Pipeline {
  MADicp icp_;
  VelEstimator vel_estimator_;
  Iso3 frame_to_map_ = isoIdentity(), keyframe_to_map_ = isoIdentity();
  V6 current_velocity_;
  std::deque<Frame*> keyframes_, frames_;
  std::vector<Iso3> trajectory_;
  Tree* current_tree_ = nullptr;
  LeafList current_leaves_;
  bool deskew_, realtime_;
  int num_keyframes_, num_threads_;
  double sensor_hz_, b_max_, p_th_, b_min_;
  size_t seq_ = 0, seq_keyframe_ = 0;
  bool is_initialized_ = false, is_map_updated_ = false;
  double last_inliers_ratio_ = 0.;

  Pipeline(double sensor_hz, bool deskew, double b_max, double rho_ker, double p_th, double b_min, double b_ratio,
           int num_keyframes, int num_threads, bool realtime)
      : icp_(b_max, rho_ker, b_ratio, num_threads), vel_estimator_(sensor_hz), deskew_(deskew), realtime_(realtime),
        num_keyframes_(num_keyframes), num_threads_(num_threads), sensor_hz_(sensor_hz), b_max_(b_max), p_th_(p_th),
        b_min_(b_min) {
    std::memset(&current_velocity_, 0, sizeof(current_velocity_));
  }
  static void freeFrame(Frame* f, bool del_tree) {
    if (del_tree) {
      delete f->tree_;
      delete f->cloud_;
    }
  }
  ~Pipeline() {
    for (Frame* f : frames_) {
      bool is_kf = std::find(keyframes_.begin(), keyframes_.end(), f) != keyframes_.end();
      if (!is_kf) { freeFrame(f, true); delete f; }
    }
    for (Frame* f : keyframes_) { freeFrame(f, true); delete f; }
  }

  // pipeline.cpp:79-123
  void deskew(Cloud* curr_cloud, const Iso3& T_prev, const Iso3& T_now) {
    const double ts = 1. / sensor_hz_;
    const Iso3 T_now_to_prev = isoMul(isoInverse(T_prev), T_now);
    const V3 w = logMapSO3(T_now_to_prev.R);
    double naive_vel[6] = {T_now_to_prev.t[0] / ts, T_now_to_prev.t[1] / ts, T_now_to_prev.t[2] / ts,
                           w[0] / ts, w[1] / ts, w[2] / ts};
    std::vector<std::pair<double, V3>> sorted(curr_cloud->size());
    for (size_t i = 0; i < sorted.size(); ++i) {
      const V3& p = (*curr_cloud)[i];
      sorted[i] = std::make_pair(std::atan2(p[1], p[0]), p);
    }
    std::sort(sorted.begin(), sorted.end(),
              [](const std::pair<double, V3>& a, const std::pair<double, V3>& b) { return a.first < b.first; });
    const double resolution = 2 * M_PI / double(CHUNKS);
    const double delta = ts / double(CHUNKS - 1);
    double t = -ts;
    auto poseAt = [&](double tt) {
      Iso3 P;
      P.R = expMapSO3(V3{{naive_vel[3] * tt, naive_vel[4] * tt, naive_vel[5] * tt}});
      P.t = V3{{naive_vel[0] * tt, naive_vel[1] * tt, naive_vel[2] * tt}};
      return P;
    };
    Iso3 meas = poseAt(t);
    double angle = M_PI - resolution;
    for (int i = int(sorted.size()) - 1; i >= 0; --i) {
      if (sorted[i].first < angle) {
        angle -= resolution;
        t += delta;
        meas = poseAt(t);
      }
      (*curr_cloud)[i] = isoApply(meas, sorted[i].second);
    }
  }

  // pipeline.cpp:267-284
  void initialize(double stamp, Cloud* cloud) {
    Frame* f = new Frame;
    f->frame_ = int(seq_);
    f->frame_to_map_ = frame_to_map_;
    f->stamp_ = stamp;
    f->cloud_ = cloud;
    f->tree_ = new Tree(cloud, 0, cloud->size(), b_max_, b_min_, 0, 0, nullptr, nullptr);
    f->tree_->getLeafs(f->leaves_);
    keyframes_.push_back(f);
    trajectory_.push_back(isoIdentity());
    is_initialized_ = true;
    is_map_updated_ = true;
    seq_++;
  }

  // pipeline.cpp:125-265
  void compute(double stamp, const double* pts, int n) {
    Cloud* cloud = new Cloud(n);
    for (int i = 0; i < n; ++i) (*cloud)[i] = V3{{pts[3 * i], pts[3 * i + 1], pts[3 * i + 2]}};
    is_map_updated_ = false;
    if (!is_initialized_) {
      initialize(stamp, cloud);
      return;
    }
    if (deskew_ && trajectory_.size() > 1)
      deskew(cloud, trajectory_[trajectory_.size() - 2], trajectory_[trajectory_.size() - 1]);
    current_tree_ = new Tree(cloud, 0, cloud->size(), b_max_, b_min_, 0, 0, nullptr, nullptr);
    current_leaves_.clear();
    current_tree_->getLeafs(current_leaves_);
    Iso3 dX;
    dX.R = expMapSO3(V3{{current_velocity_.v[3] * 1. / sensor_hz_, current_velocity_.v[4] * 1. / sensor_hz_,
                         current_velocity_.v[5] * 1. / sensor_hz_}});
    dX.t = V3{{current_velocity_.v[0] * 1. / sensor_hz_, current_velocity_.v[1] * 1. / sensor_hz_,
               current_velocity_.v[2] * 1. / sensor_hz_}};
    const Iso3 prediction = isoMul(frame_to_map_, dX);
    icp_.setMoving(current_leaves_);
    icp_.init(prediction);
    std::vector<Tree*> kfs;
    for (Frame* f : keyframes_) kfs.push_back(f->tree_);
    icp_loop(icp_, kfs, current_leaves_, MAX_ICP_ITS, num_threads_, nullptr, false);  // :166-193, realtime off
    frame_to_map_ = icp_.X_;
    int matched_leaves = 0;
    for (Tree* l : current_leaves_) matched_leaves += l->matched_ ? 1 : 0;
    const double inliers_ratio = double(matched_leaves) / double(current_leaves_.size());
    last_inliers_ratio_ = inliers_ratio;
    trajectory_.push_back(frame_to_map_);
    std::vector<Iso3> odom_window;
    for (int i = std::max(0, int(trajectory_.size()) - SMOOTHING_T); i < int(trajectory_.size()); ++i)
      odom_window.push_back(trajectory_[i]);
    vel_estimator_.init(current_velocity_);
    vel_estimator_.setOdometry(odom_window);
    vel_estimator_.oneRound();
    current_velocity_ = vel_estimator_.X_;
    Frame* cur = new Frame;
    cur->frame_ = int(seq_);
    cur->frame_to_map_ = frame_to_map_;
    cur->stamp_ = stamp;
    cur->weight_ = inverseDeterminant6(icp_.H_adder_);
    current_tree_->applyTransform(frame_to_map_.R, frame_to_map_.t);
    cur->tree_ = current_tree_;
    cur->cloud_ = cloud;
    cur->leaves_ = current_leaves_;
    frames_.push_back(cur);
    if (frames_.size() > size_t(FRAME_WINDOW)) {
      freeFrame(frames_.front(), true);
      delete frames_.front();
      frames_.pop_front();
    }
    if (inliers_ratio < p_th_) {
      double best_weight = std::numeric_limits<double>::max();
      int new_seq = 0;
      Frame* best_frame = nullptr;
      for (Frame* f : frames_)
        if (f->weight_ < best_weight) {
          best_weight = f->weight_;
          new_seq = f->frame_;
          best_frame = f;
        }
      while (!frames_.empty() && frames_.front()->frame_ <= new_seq) {
        if (frames_.front()->frame_ < new_seq) {
          freeFrame(frames_.front(), true);
          delete frames_.front();
        }
        frames_.pop_front();
      }
      keyframes_.push_back(best_frame);
      if (keyframes_.size() > size_t(num_keyframes_)) {
        freeFrame(keyframes_.front(), true);
        delete keyframes_.front();
        keyframes_.pop_front();
      }
      is_map_updated_ = true;
      seq_keyframe_ = size_t(new_seq);
      keyframe_to_map_ = best_frame->frame_to_map_;
    }
    seq_++;
  }
};

}  // namespace orc
