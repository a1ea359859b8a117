// mloam_shim.hpp — C++ host side above the C ABI (include/mloam_b200.h): the reference's class surface for the
// hot path, so that L4/L4' code (Estimator, lidar_mapper process()) keeps compiling against the same names,
// argument meaning and error behaviour while the work runs in the sm_90a kernels.
//
//   reference type / function                                       here
//   common::PointI, PointICloud (type.h:20-23)                      common::PointI, common::PointICloud (POD stand-ins
//                                                                    when PCL is absent; with -DMLOAM_WITH_PCL the pcl types)
//   ScanInfo, cloudFeature, PointPlaneFeature (parameters.h:161-207) same names, same members
//   Pose (pose.h)                                                   Pose { q_ (x,y,z,w), t_ } minimal
//   FeatureExtract (feature_extract.hpp:55-129)                     same method names / argument order
//   pcl::KdTreeFLANN<PointType>::Ptr                                mloam::MapHandle (setInputCloud -> mloam_map_build)
//   PoseLocalParameterization (pose_local_parameterization.h)        Plus / ComputeJacobian / GlobalSize / LocalSize /
//                                                                    setParameter / is_degenerate_ / V_update_
//   LidarMap{PlaneNorm,Edge}Factor, LidarScan{PlaneNorm,Edge,EdgeVector}Factor, LidarPureOdom{PlaneNorm,Edge}Factor,
//   LidarOnlineCalib{PlaneNorm,Edge}Factor                          same ctor arguments, bool Evaluate(param, residuals, jacobians)
//   LidarTracker::trackCloud (lidar_tracker.h:48)                   same signature
//   scan2MapOptimization (lidar_mapper_keyframe.cpp:423)            mloam::scan2MapOptimization(...)
//
// Error conventions follow the reference: Evaluate / Plus return true; too few correspondences is not an error
// (the pose is returned unchanged); a CUDA/ABI failure — which has no counterpart in the reference — throws
// std::runtime_error with mloam_last_error().  There is no CPU fallback anywhere in this header.
// Contexts: one per host thread (thread_local), matching the reference's one-OpenMP-thread-per-LiDAR use
// (estimator.cpp:249,423).
#pragma once
#include <array>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "mloam_context.hpp"
#include "mloam_io.hpp"

// ----------------------------------------------------------------------------------------------- point types
namespace common {
#ifndef MLOAM_WITH_PCL
struct PointI {
  float x, y, z, intensity;
};
template <typename P>
struct PointCloudT {
  std::vector<P> points;
  size_t size() const { return points.size(); }
  bool empty() const { return points.empty(); }
  void clear() { points.clear(); }
  void push_back(const P &p) { points.push_back(p); }
  void resize(size_t n) { points.resize(n); }
  P &operator[](size_t i) { return points[i]; }
  const P &operator[](size_t i) const { return points[i]; }
  typename std::vector<P>::const_iterator begin() const { return points.begin(); }
  typename std::vector<P>::const_iterator end() const { return points.end(); }
  PointCloudT &operator+=(const PointCloudT &o) {
    points.insert(points.end(), o.points.begin(), o.points.end());
    return *this;
  }
};
typedef PointCloudT<PointI> PointICloud;
#endif
}  // namespace common

static_assert(sizeof(common::PointI) == sizeof(mloam_point_t) || sizeof(common::PointI) == 32,
              "PointI must be the 16 B payload or pcl::PointXYZI (32 B)");

// estimator/src/estimator/parameters.h:192-207
class ScanInfo {
 public:
  ScanInfo(const int &n_scan, const bool &segment_flag) {
    segment_flag_ = segment_flag;
    scan_start_ind_.resize(n_scan);
    scan_end_ind_.resize(n_scan);
    ground_flag_.clear();
  }
  std::vector<int> scan_start_ind_, scan_end_ind_;
  bool segment_flag_;
  std::vector<bool> ground_flag_;
};

// parameters.h:161
typedef std::map<std::string, common::PointICloud> cloudFeature;

// Minimal Pose (estimator/src/estimator/pose.h): q_ = (x, y, z, w), normalised on construction (pose.cpp:34-41).
struct Pose {
  std::array<double, 4> q_{{0, 0, 0, 1}};
  std::array<double, 3> t_{{0, 0, 0}};
  Pose() {}
  Pose(const std::array<double, 4> &q, const std::array<double, 3> &t) : q_(q), t_(t) {
    const double n = std::sqrt(q_[0] * q_[0] + q_[1] * q_[1] + q_[2] * q_[2] + q_[3] * q_[3]);
    for (double &v : q_) v /= n;
  }
  void toParam(double *x) const {  // [tx ty tz qx qy qz qw], pose_local_parameterization.h:20
    x[0] = t_[0], x[1] = t_[1], x[2] = t_[2], x[3] = q_[0], x[4] = q_[1], x[5] = q_[2], x[6] = q_[3];
  }
  static Pose fromParam(const double *x) { return Pose({{x[3], x[4], x[5], x[6]}}, {{x[0], x[1], x[2]}}); }
};

// parameters.h:163-175 (Eigen members replaced by fixed arrays; coeffs_: 4 used for 's', 6 for 'c')
class PointPlaneFeature {
 public:
  PointPlaneFeature() : idx_(0), laser_idx_(0), type_('n') {}
  size_t idx_;
  size_t laser_idx_;
  std::array<double, 3> point_{{0, 0, 0}};
  std::array<double, 6> coeffs_{{0, 0, 0, 0, 0, 0}};
  std::array<double, 6> jaco_{{0, 0, 0, 0, 0, 0}};
  char type_;
};

namespace mloam {

inline std::vector<mloam_point_t> pack(const common::PointICloud &c) {
  std::vector<mloam_point_t> v(c.size());
  for (size_t i = 0; i < c.size(); i++) v[i] = mloam_point_t{c.points[i].x, c.points[i].y, c.points[i].z, c.points[i].intensity};
  return v;
}
inline void unpack(const mloam_point_t *p, int n, common::PointICloud &c) {
  c.clear();
  c.resize((size_t)n);
  for (int i = 0; i < n; i++) {
    c.points[i].x = p[i].x, c.points[i].y = p[i].y, c.points[i].z = p[i].z, c.points[i].intensity = p[i].intensity;
  }
}

// Stand-in for pcl::KdTreeFLANN<PointType>::Ptr: a map slot in the calling thread's context.
class MapHandle {
 public:
  explicit MapHandle(int slot, float cell = 0.f) : slot_(slot), cell_(cell) {}
  void setInputCloud(const common::PointICloud &cloud) {  // KdTreeFLANN::setInputCloud
    std::vector<mloam_point_t> v = pack(cloud);
    check(ThreadContext::get(), mloam_map_build(ThreadContext::get(), slot_, v.data(), (int)v.size(), cell_), "mloam_map_build");
  }
  // KdTreeFLANN::nearestKSearch (K in {1,5,10}; neighbours beyond `max_sqdist` are reported as -1 / inf)
  int nearestKSearch(const common::PointI &p, int k, std::vector<int> &idx, std::vector<float> &sqd, float max_sqdist = 1.0f) const {
    idx.assign(k, -1);
    sqd.assign(k, INFINITY);
    mloam_point_t q{p.x, p.y, p.z, p.intensity};
    check(ThreadContext::get(), mloam_knn(ThreadContext::get(), slot_, &q, 1, nullptr, k, max_sqdist, idx.data(), sqd.data()), "mloam_knn");
    int got = 0;
    while (got < k && idx[got] >= 0) got++;
    return got;
  }
  int slot() const { return slot_; }

 private:
  int slot_;
  float cell_;
};
typedef std::shared_ptr<MapHandle> MapHandlePtr;

}  // namespace mloam

// ----------------------------------------------------------------------------------------------- FeatureExtract
class FeatureExtract {
 public:
  FeatureExtract() {}

  // feature_extract.cpp:118-297
  void extractCloud(const common::PointICloud &laser_cloud_in, const ScanInfo &scan_info, cloudFeature &cloud_feature) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> in = mloam::pack(laser_cloud_in);
    const int n = (int)in.size();
    std::vector<mloam_point_t> b0(n + 1), b1(n + 1), b2(n + 1), b3(n + 1);
    mloam_features_t f;
    f.corner_points_sharp = b0.data(), f.corner_points_less_sharp = b1.data();
    f.surf_points_flat = b2.data(), f.surf_points_less_flat = b3.data();
    f.cap = n;
    mloam::check(ctx, mloam_extract_features(ctx, in.data(), n, scan_info.scan_start_ind_.data(), scan_info.scan_end_ind_.data(),
                                             (int)scan_info.scan_start_ind_.size(), &f), "mloam_extract_features");
    cloud_feature.clear();
    cloud_feature["laser_cloud"] = laser_cloud_in;  // :281-285
    mloam::unpack(b0.data(), f.n_sharp, cloud_feature["corner_points_sharp"]);
    mloam::unpack(b1.data(), f.n_less_sharp, cloud_feature["corner_points_less_sharp"]);
    mloam::unpack(b2.data(), f.n_flat, cloud_feature["surf_points_flat"]);
    mloam::unpack(b3.data(), f.n_less_flat, cloud_feature["surf_points_less_flat"]);
  }

  // feature_extract.hpp:378-643.  The kd-tree argument is the map handle the cloud was loaded into; `cloud_map`
  // is kept in the signature for source compatibility (the device copy is used).
  void matchCornerFromMap(const mloam::MapHandlePtr &kdtree_corner_from_map, const common::PointICloud &cloud_map,
                          const common::PointICloud &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features,
                          const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    matchFromMap('c', kdtree_corner_from_map, cloud_map, cloud_data, pose_local, features, N_NEIGH, CHECK_FOV);
  }
  void matchSurfFromMap(const mloam::MapHandlePtr &kdtree_surf_from_map, const common::PointICloud &cloud_map,
                        const common::PointICloud &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features,
                        const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    matchFromMap('s', kdtree_surf_from_map, cloud_map, cloud_data, pose_local, features, N_NEIGH, CHECK_FOV);
  }
  // feature_extract.hpp:645-883 (per-point forms)
  bool matchCornerPointFromMap(const mloam::MapHandlePtr &kd, const common::PointICloud &cloud_map, const common::PointI &point_ori,
                               const Pose &pose_local, PointPlaneFeature &feature, const size_t &idx, const size_t &N_NEIGH = 5,
                               const bool &CHECK_FOV = true) {
    return matchPointFromMap('c', kd, cloud_map, point_ori, pose_local, feature, idx, N_NEIGH, CHECK_FOV);
  }
  bool matchSurfPointFromMap(const mloam::MapHandlePtr &kd, const common::PointICloud &cloud_map, const common::PointI &point_ori,
                             const Pose &pose_local, PointPlaneFeature &feature, const size_t &idx, const size_t &N_NEIGH = 5,
                             const bool &CHECK_FOV = true) {
    return matchPointFromMap('s', kd, cloud_map, point_ori, pose_local, feature, idx, N_NEIGH, CHECK_FOV);
  }
  // feature_extract.hpp:131-376
  void matchCornerFromScan(const mloam::MapHandlePtr &kd, const common::PointICloud &cloud_scan, const common::PointICloud &cloud_data,
                           const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    matchFromScan('c', kd, cloud_scan, cloud_data, pose_local, features);
  }
  void matchSurfFromScan(const mloam::MapHandlePtr &kd, const common::PointICloud &cloud_scan, const common::PointICloud &cloud_data,
                         const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    matchFromScan('s', kd, cloud_scan, cloud_data, pose_local, features);
  }

 private:
  void matchFromMap(char type, const mloam::MapHandlePtr &kd, const common::PointICloud &, const common::PointICloud &cloud_data,
                    const Pose &pose_local, std::vector<PointPlaneFeature> &features, size_t n_neigh, bool check_fov) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    mloam_params_t &P = mloam::ThreadContext::params();
    P.n_neigh = (int)n_neigh, P.check_fov = check_fov ? 1 : 0;
    mloam::ThreadContext::applyParams();
    std::vector<mloam_point_t> q = mloam::pack(cloud_data);
    const int n = (int)q.size();
    std::vector<unsigned char> valid(n + 1);
    std::vector<double> coeffs((size_t)n * 6 + 6);
    double x[7];
    pose_local.toParam(x);
    mloam::check(ctx, mloam_match_from_map(ctx, kd->slot(), type, q.data(), n, x, valid.data(), coeffs.data(), nullptr),
                 "mloam_match_from_map");
    features.clear();  // compacted in query order (:398-399, :536-537)
    for (int i = 0; i < n; i++) {
      if (!valid[i]) continue;
      PointPlaneFeature f;
      f.idx_ = (size_t)i;
      f.point_ = {{(double)q[i].x, (double)q[i].y, (double)q[i].z}};
      for (int k = 0; k < 6; k++) f.coeffs_[k] = coeffs[(size_t)i * 6 + k];
      f.laser_idx_ = (size_t)q[i].intensity;
      f.type_ = type;
      features.push_back(f);
    }
  }
  bool matchPointFromMap(char type, const mloam::MapHandlePtr &kd, const common::PointICloud &map, const common::PointI &p, const Pose &pose,
                         PointPlaneFeature &feature, size_t idx, size_t n_neigh, bool check_fov) {
    common::PointICloud one;
    one.push_back(p);
    std::vector<PointPlaneFeature> fs;
    matchFromMap(type, kd, map, one, pose, fs, n_neigh, check_fov);
    if (fs.empty()) return false;
    feature = fs[0];
    feature.idx_ = idx;
    return true;
  }
  void matchFromScan(char type, const mloam::MapHandlePtr &kd, const common::PointICloud &, const common::PointICloud &cloud_data,
                     const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> q = mloam::pack(cloud_data);
    const int n = (int)q.size();
    std::vector<unsigned char> valid(n + 1);
    std::vector<double> coeffs((size_t)n * 6 + 6);
    double x[7];
    pose_local.toParam(x);
    mloam::check(ctx, mloam_match_from_scan(ctx, kd->slot(), type, q.data(), n, x, valid.data(), coeffs.data(), nullptr),
                 "mloam_match_from_scan");
    features.clear();
    for (int i = 0; i < n; i++) {
      if (!valid[i]) continue;
      PointPlaneFeature f;
      f.idx_ = (size_t)i;
      f.point_ = {{(double)q[i].x, (double)q[i].y, (double)q[i].z}};
      for (int k = 0; k < 6; k++) f.coeffs_[k] = coeffs[(size_t)i * 6 + k];
      f.type_ = type == 's' ? 's' : 'n';  // the reference leaves type_ at 'n' for scan corners (:262-266)
      features.push_back(f);
    }
  }
};

// ----------------------------------------------------------------------------------------------- parameterisation
// pose_local_parameterization.{h,cpp}.  With Ceres present derive from ceres::LocalParameterization (same virtuals).
class PoseLocalParameterization {
 public:
  PoseLocalParameterization() { setParameter(); }
  virtual ~PoseLocalParameterization() {}
  virtual bool Plus(const double *x, const double *delta, double *x_plus_delta) const {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    mloam::check(ctx, mloam_pose_plus(ctx, x, delta, V_update_.data(), x_plus_delta), "mloam_pose_plus");
    return true;
  }
  virtual bool ComputeJacobian(const double *, double *jacobian) const {  // 7x6 row-major [I6; 0] (.cpp:50-56)
    for (int i = 0; i < 42; i++) jacobian[i] = 0.0;
    for (int i = 0; i < 6; i++) jacobian[i * 6 + i] = 1.0;
    return true;
  }
  virtual int GlobalSize() const { return 7; }
  virtual int LocalSize() const { return 6; }
  void setParameter() {
    is_degenerate_ = false;
    for (int i = 0; i < 36; i++) V_update_[i] = (i % 7 == 0) ? 1.0 : 0.0;
  }
  bool is_degenerate_;
  std::array<double, 36> V_update_;  // row-major 6x6 (Eigen::Matrix<double,6,6> in the reference)
};

// ----------------------------------------------------------------------------------------------- factors
namespace mloam {
// Shared implementation: one factor = one batch of size 1 through mloam_factor_evaluate.
class FactorBase {
 public:
  FactorBase(int kind, const double *point3, const double *coeffs, int n_coeff, double sqrt_info) : kind_(kind), sqrt_info_(sqrt_info) {
    for (int k = 0; k < 3; k++) point_[k] = point3[k];
    for (int k = 0; k < 6; k++) coeff_[k] = k < n_coeff ? coeffs[k] : 0.0;
  }
  virtual ~FactorBase() {}
  // ceres::CostFunction::Evaluate: null-tolerant on `jacobians` and on each jacobians[k]
  bool Evaluate(double const *const *param, double *residuals, double **jacobians) const {
    mloam_ctx_t *ctx = ThreadContext::get();
    const int nblk = kind_ >= 3 ? 3 : 1, rows = kind_ == 2 ? 3 : 1;
    double x[21];
    for (int b = 0; b < nblk; b++) std::memcpy(x + 7 * b, param[b], 7 * sizeof(double));
    double J[63];
    check(ctx, mloam_factor_evaluate(ctx, kind_, 1, point_, coeff_, &sqrt_info_, x, residuals, jacobians ? J : nullptr),
          "mloam_factor_evaluate");
    if (jacobians) {
      if (nblk == 1) {
        if (jacobians[0]) std::memcpy(jacobians[0], J, sizeof(double) * rows * 7);
      } else {
        for (int b = 0; b < 3; b++)
          if (jacobians[b]) std::memcpy(jacobians[b], J + 7 * b, sizeof(double) * 7);
      }
    }
    return true;
  }

 protected:
  int kind_;
  double point_[3], coeff_[6], sqrt_info_;
};
inline double map_sqrt_info(double cov_trace) {  // lidar_map_factor.hpp:34,41
  const double s = std::sqrt(1.0 / cov_trace);
  return s >= 3.0 ? 1.0 : s / 3.0;
}
}  // namespace mloam

// lidar_map_factor.hpp:26-126 / :130-235  (cov_matrix argument reduced to its trace, which is all the factor uses)
class LidarMapPlaneNormFactor : public mloam::FactorBase {
 public:
  LidarMapPlaneNormFactor(const double point[3], const double coeff[4], double cov_trace = 3.0)
      : FactorBase(0, point, coeff, 4, mloam::map_sqrt_info(cov_trace)) {}
};
class LidarMapEdgeFactor : public mloam::FactorBase {
 public:
  LidarMapEdgeFactor(const double point[3], const double coeff[6], double cov_trace = 3.0)
      : FactorBase(1, point, coeff, 6, mloam::map_sqrt_info(cov_trace)) {}
};
// lidar_scan_factor.hpp:25-126 / :130-232 / :236-343 (s = 1: the distortion slerp is the identity)
class LidarScanPlaneNormFactor : public mloam::FactorBase {
 public:
  LidarScanPlaneNormFactor(const double point[3], const double coeff[4], const double &s = 1.0) : FactorBase(0, point, coeff, 4, 1.0) { (void)s; }
};
class LidarScanEdgeFactor : public mloam::FactorBase {
 public:
  LidarScanEdgeFactor(const double point[3], const double coeff[6], const double &s = 1.0) : FactorBase(1, point, coeff, 6, 1.0) { (void)s; }
};
class LidarScanEdgeFactorVector : public mloam::FactorBase {
 public:
  LidarScanEdgeFactorVector(const double point[3], const double coeff[6], const double &s = 1.0) : FactorBase(2, point, coeff, 6, 1.0) { (void)s; }
};
// lidar_pure_odom_factor.hpp:27-195 / :198-381 — parameter blocks (pivot, pose_i, ext)
class LidarPureOdomPlaneNormFactor : public mloam::FactorBase {
 public:
  LidarPureOdomPlaneNormFactor(const double point[3], const double coeff[4], const double &sqrt_info = 1.0)
      : FactorBase(3, point, coeff, 4, sqrt_info) {}
};
class LidarPureOdomEdgeFactor : public mloam::FactorBase {
 public:
  LidarPureOdomEdgeFactor(const double point[3], const double coeff[6], const double &sqrt_info = 1.0)
      : FactorBase(4, point, coeff, 6, sqrt_info) {}
};
// lidar_online_calib_factor.hpp:24-121 / :125-227 — same algebra as the map factors with T = ext and sqrt_info direct
class LidarOnlineCalibPlaneNormFactor : public mloam::FactorBase {
 public:
  LidarOnlineCalibPlaneNormFactor(const double point[3], const double coeff[4], const double &sqrt_info = 1.0)
      : FactorBase(0, point, coeff, 4, sqrt_info) {}
};
class LidarOnlineCalibEdgeFactor : public mloam::FactorBase {
 public:
  LidarOnlineCalibEdgeFactor(const double point[3], const double coeff[6], const double &sqrt_info = 1.0)
      : FactorBase(1, point, coeff, 6, sqrt_info) {}
};

// ----------------------------------------------------------------------------------------------- LidarTracker
// lidar_tracker.h:44-52
class LidarTracker {
 public:
  LidarTracker() {}
  Pose trackCloud(const cloudFeature &prev_cloud_feature, const cloudFeature &cur_cloud_feature, const Pose &pose_ini) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> a = mloam::pack(prev_cloud_feature.find("corner_points_less_sharp")->second);
    std::vector<mloam_point_t> b = mloam::pack(prev_cloud_feature.find("surf_points_less_flat")->second);
    std::vector<mloam_point_t> c = mloam::pack(cur_cloud_feature.find("corner_points_sharp")->second);
    std::vector<mloam_point_t> d = mloam::pack(cur_cloud_feature.find("surf_points_flat")->second);
    double x[7], y[7];
    pose_ini.toParam(x);
    mloam::check(ctx, mloam_track_cloud(ctx, a.data(), (int)a.size(), b.data(), (int)b.size(), c.data(), (int)c.size(), d.data(),
                                        (int)d.size(), x, y, nullptr), "mloam_track_cloud");
    return Pose::fromParam(y);
  }
  FeatureExtract f_extract_;
};

// ----------------------------------------------------------------------------------------------- good features
// ActiveFeatureSelection::goodFeatureMatching (lidar_mapper.h:229-573).  The kd-tree argument of the reference is the
// map slot here (MLOAM_MAP_SURF / MLOAM_MAP_CORNER, built with MapHandle or scan2MapOptimization); gf_method is the
// reference's string.  sub_mat_H comes back as the reference leaves it.  The seed replaces std::random_device.
class ActiveFeatureSelection {
 public:
  unsigned long long seed = 0;
  void goodFeatureMatching(int map_slot, const common::PointICloud &laser_cloud, const Pose &pose_local, std::vector<size_t> &sel_feature_idx,
                           const char feature_type, const std::string &gf_method, const double gf_ratio, double sub_mat_H[36],
                           const float *cov_vec6 = nullptr) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    // gd_fix / gd_float are one selection; gd_float's ratio policy (lidar_mapper_keyframe.cpp:456-495) is mloam_set_gf_float
    const int method = gf_method == "wo_gf" ? 0 : gf_method == "rnd" ? 1 : gf_method == "fps" ? 2 : 3;
    std::vector<mloam_point_t> pts = mloam::pack(laser_cloud);
    std::vector<int> sel(pts.size() + 1);
    int n_sel = 0;
    double x[7];
    pose_local.toParam(x);
    mloam::check(ctx, mloam_good_features(ctx, map_slot, feature_type, pts.data(), (int)pts.size(), cov_vec6, x, method, gf_ratio, seed++,
                                          sel.data(), &n_sel, sub_mat_H, nullptr, nullptr), "mloam_good_features");
    sel_feature_idx.assign(sel.begin(), sel.begin() + n_sel);
  }
  // ActiveFeatureSelection::evalFullHessian (lidar_mapper.h:176-227): mat_H (row-major 6x6) and feat_num accumulate, as in the reference
  void evalFullHessian(int map_slot, const common::PointICloud &laser_cloud, const Pose &pose_local, const char feature_type, double mat_H[36],
                       int &feat_num, const float *cov_vec6 = nullptr) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> pts = mloam::pack(laser_cloud);
    double x[7];
    pose_local.toParam(x);
    mloam::check(ctx, mloam_full_hessian(ctx, map_slot, feature_type, pts.data(), (int)pts.size(), cov_vec6, x, mat_H, &feat_num), "mloam_full_hessian");
  }
};

// ----------------------------------------------------------------------------------------------- mapper entry
namespace mloam {
// scan2MapOptimization (lidar_mapper_keyframe.cpp:423-639): the two submaps are (re)built with setInputCloud every
// call, exactly as the reference does; returns false when the map-size gate (:429) rejects the frame.
inline bool scan2MapOptimization(const common::PointICloud &laser_cloud_surf_from_map, const common::PointICloud &laser_cloud_corner_from_map,
                                 const common::PointICloud &laser_cloud_surf, const common::PointICloud &laser_cloud_corner, Pose &pose_wmap_curr,
                                 mloam_solve_stats_t *stats = nullptr) {
  mloam_ctx_t *ctx = ThreadContext::get();
  std::vector<mloam_point_t> sm = pack(laser_cloud_surf_from_map), cm = pack(laser_cloud_corner_from_map);
  check(ctx, mloam_map_build(ctx, MLOAM_MAP_SURF, sm.data(), (int)sm.size(), 0.f), "mloam_map_build(surf)");
  check(ctx, mloam_map_build(ctx, MLOAM_MAP_CORNER, cm.data(), (int)cm.size(), 0.f), "mloam_map_build(corner)");
  std::vector<mloam_point_t> ss = pack(laser_cloud_surf), cs = pack(laser_cloud_corner);
  double x[7], y[7];
  pose_wmap_curr.toParam(x);
  mloam_solve_stats_t st;
  check(ctx, mloam_scan2map(ctx, ss.data(), (int)ss.size(), cs.data(), (int)cs.size(), x, y, &st), "mloam_scan2map");
  if (stats) *stats = st;
  if (st.ran) {  // double2Vector (:247-252): no normalisation
    pose_wmap_curr.t_ = {{y[0], y[1], y[2]}};
    pose_wmap_curr.q_ = {{y[3], y[4], y[5], y[6]}};
  }
  return st.ran != 0;
}
}  // namespace mloam

// ----------------------------------------------------------------------------------------------- DISTORTION
namespace mloam {
// The pose_undist of Estimator::process (estimator.cpp:575-579) and the per-LiDAR choice of undistortMeasurements (:376-408), for
// mloam_frame_undistort: pose_ext[n]^-1 * pose_rlt * pose_ext[n], every LiDAR taking idx_ref's unless estimate_extrinsic == 2.
inline std::vector<Pose> undistortPoses(const Pose &pose_rlt, int idx_ref, const std::vector<Pose> &pose_ext, int estimate_extrinsic) {
  std::vector<double> e(7 * pose_ext.size()), out(7 * pose_ext.size());
  for (size_t n = 0; n < pose_ext.size(); n++) pose_ext[n].toParam(&e[7 * n]);
  double r[7];
  pose_rlt.toParam(r);
  if (mloam_undistort_poses(r, idx_ref, (int)pose_ext.size(), e.data(), estimate_extrinsic, out.data()) != MLOAM_OK)
    throw std::runtime_error("mloam_undistort_poses: invalid arguments");
  std::vector<Pose> res(pose_ext.size());
  for (size_t n = 0; n < pose_ext.size(); n++) {
    const double *o = &out[7 * n];
    res[n].t_ = {{o[0], o[1], o[2]}}, res[n].q_ = {{o[3], o[4], o[5], o[6]}};  // as computed: already normalised
  }
  return res;
}
// mloam_set_distortion / mloam_frame_undistort / mloam_frame_set_next_undistort on ctx, the context that runs the frames (the poses as
// undistortPoses returns them)
inline void setDistortion(mloam_ctx_t *ctx, bool on, float scan_period) {
  check(ctx, mloam_set_distortion(ctx, on ? 1 : 0, scan_period), "mloam_set_distortion");
}
inline void undistortMeasurements(mloam_ctx_t *ctx, const std::vector<Pose> &pose_undist) {
  std::vector<double> x(7 * pose_undist.size());
  for (size_t l = 0; l < pose_undist.size(); l++) pose_undist[l].toParam(&x[7 * l]);
  check(ctx, mloam_frame_undistort(ctx, (int)pose_undist.size(), x.data()), "mloam_frame_undistort");
}
// the poses of the sweep announced by the last mloam_frame_set_next* call: the look-ahead undistorts it too
inline void undistortMeasurementsNext(mloam_ctx_t *ctx, const std::vector<Pose> &pose_undist) {
  std::vector<double> x(7 * pose_undist.size());
  for (size_t l = 0; l < pose_undist.size(); l++) pose_undist[l].toParam(&x[7 * l]);
  check(ctx, mloam_frame_set_next_undistort(ctx, (int)pose_undist.size(), x.data()), "mloam_frame_set_next_undistort");
}
}  // namespace mloam

// ----------------------------------------------------------------------------------------------- pubPointCloud
namespace mloam {
// mloam_set_registered / mloam_frame_registered on ctx: laser_cloud_full_res (with the outlier points when the outlier cloud is on),
// laser_cloud_surf_last and laser_cloud_corner_last of the last mloam_frame* call, moved into the world frame with pose_wmap_curr
// (lidar_mapper_keyframe.cpp:690-714)
inline void setRegistered(mloam_ctx_t *ctx, bool on) { check(ctx, mloam_set_registered(ctx, on ? 1 : 0), "mloam_set_registered"); }
inline void frameRegistered(mloam_ctx_t *ctx, int which, common::PointICloud &out) {
  int n = 0;
  check(ctx, mloam_frame_registered(ctx, which, nullptr, 0, &n), "mloam_frame_registered");
  std::vector<mloam_point_t> pts((size_t)n);
  check(ctx, mloam_frame_registered(ctx, which, pts.data(), n, &n), "mloam_frame_registered");
  unpack(pts.data(), n, out);
}
inline void frameRegistered(mloam_ctx_t *ctx, common::PointICloud &full_res, common::PointICloud &surf_last, common::PointICloud &corner_last) {
  frameRegistered(ctx, MLOAM_REGISTERED_FULL_RES, full_res);
  frameRegistered(ctx, MLOAM_REGISTERED_SURF, surf_last);
  frameRegistered(ctx, MLOAM_REGISTERED_CORNER, corner_last);
}
}  // namespace mloam

// ----------------------------------------------------------------------------------------------- PointCloud2 messages
namespace mloam {
// laserCloudHandler -> mloam_frame_msg: the rig's messages as the driver nodes receive them (one per LiDAR, the order of mloam_set_lidars).
// setFrontEndLayout resolves each driver's layout once (lane 3: "timestamp" with time_field 1, none otherwise); frameMsg runs the frame on
// the messages' bytes, which the library unpacks on the device (the maps are the frame's submaps, rebuilt as mloam_frame_raw does).
inline void setFrontEndLayout(mloam_ctx_t *ctx, const std::vector<io::PointCloud2View> &msgs, bool time_field) {
  std::vector<mloam_pc2_layout_t> layouts(msgs.size());
  for (size_t l = 0; l < msgs.size(); l++)
    if (!io::resolvePointCloud2Layout(msgs[l], time_field ? "timestamp" : nullptr, layouts[l]))
      throw std::runtime_error("setFrontEndLayout: a message lacks x / y / z (or timestamp) as FLOAT32 / FLOAT64 fields inside the point");
  check(ctx, mloam_set_front_end_layout(ctx, (int)layouts.size(), layouts.data()), "mloam_set_front_end_layout");
}
inline bool frameMsg(mloam_ctx_t *ctx, const std::vector<io::PointCloud2View> &msgs, const common::PointICloud &laser_cloud_surf_from_map,
                     const common::PointICloud &laser_cloud_corner_from_map, Pose &pose_wmap_curr, mloam_solve_stats_t *stats = nullptr) {
  std::vector<mloam_pc2_msg_t> m(msgs.size());
  for (size_t l = 0; l < msgs.size(); l++) m[l] = io::pointCloud2Msg(msgs[l]);
  std::vector<mloam_point_t> sm = pack(laser_cloud_surf_from_map), cm = pack(laser_cloud_corner_from_map);
  double x[7], y[7];
  pose_wmap_curr.toParam(x);
  mloam_solve_stats_t st;
  check(ctx, mloam_frame_msg(ctx, m.data(), sm.data(), (int)sm.size(), cm.data(), (int)cm.size(), 1, x, y, &st), "mloam_frame_msg");
  if (stats) *stats = st;
  if (st.ran) {
    pose_wmap_curr.t_ = {{y[0], y[1], y[2]}};
    pose_wmap_curr.q_ = {{y[3], y[4], y[5], y[6]}};
  }
  return st.ran != 0;
}
}  // namespace mloam

// ----------------------------------------------------------------------------------------------- published clouds as PointCloud2
namespace mloam {
// pcl::toROSMsg of the clouds pubPointCloud (lidar_mapper_keyframe.cpp:690-714) and pubGlobalMap (:780-851) publish, packed on the
// device by one launch: sources[k] (MLOAM_MSG_*) into storage[k], which the returned views point at.  Keep the storage from call to
// call, so that its capacity is reused.
inline std::vector<io::PointCloud2View> cloudMsgs(mloam_ctx_t *ctx, const std::vector<int> &sources, std::vector<std::vector<uint8_t>> &storage) {
  storage.resize(sources.size());
  std::vector<std::vector<uint8_t> *> data;
  for (auto &s : storage) data.push_back(&s);
  std::vector<int> width;
  check(ctx, io::cloudMsgs(ctx, sources, data, width), "mloam_cloud_msgs");
  std::vector<io::PointCloud2View> views;
  for (size_t k = 0; k < sources.size(); k++) views.push_back(io::cloudMsgView(sources[k], (size_t)width[k], storage[k].data()));
  return views;
}
}  // namespace mloam

// ---- Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 over the whole rig (estimator.cpp:633-642, 670-787): mloam_calib_rig on ctx.
// surf[n] / corner[n]: LiDAR n's features (sensor frame); pose_i and pose_ext (one per LiDAR, pose_ext[idx_ref] constant) in/out; prior
// (nullable): the PriorFactor targets tbl_ / qbl_ with prior_pos / prior_rot (prior_factor.hpp:27-72).  rows (nullable): each LiDAR's
// feature rows of the last evaluation.
namespace mloam {
inline mloam_solve_stats_t calibRig(mloam_ctx_t *ctx, int idx_ref, const std::vector<common::PointICloud> &surf, const std::vector<common::PointICloud> &corner,
                                    const Pose &pose_pivot, Pose &pose_i, std::vector<Pose> &pose_ext, const std::vector<Pose> *prior, double prior_pos,
                                    double prior_rot, int max_outer, int max_inner, bool own_cal_maps = false, std::vector<int> *rows = nullptr,
                                    double huber_a = 1.0) {
  const size_t L = pose_ext.size();
  if (surf.size() != L || corner.size() != L || (prior && prior->size() != L)) throw std::invalid_argument("calibRig: one cloud / prior per LiDAR");
  std::vector<mloam_point_t> s, c;
  std::vector<int> ns(L), nc(L), r(L);
  for (size_t n = 0; n < L; n++) {
    const std::vector<mloam_point_t> a = pack(surf[n]), b = pack(corner[n]);
    s.insert(s.end(), a.begin(), a.end()), c.insert(c.end(), b.begin(), b.end());
    ns[n] = (int)a.size(), nc[n] = (int)b.size();
  }
  std::vector<double> ext(7 * L), pr(prior ? 7 * L : 0);
  for (size_t n = 0; n < L; n++) {
    pose_ext[n].toParam(&ext[7 * n]);
    if (prior) (*prior)[n].toParam(&pr[7 * n]);
  }
  double pv[7], pi[7];
  pose_pivot.toParam(pv), pose_i.toParam(pi);
  mloam_solve_stats_t st;
  check(ctx, mloam_calib_rig(ctx, (int)L, idx_ref, s.data(), ns.data(), c.data(), nc.data(), pv, pi, ext.data(), prior ? pr.data() : nullptr,
                             prior ? prior_pos : 0.0, prior ? prior_rot : 0.0, max_outer, max_inner, huber_a, own_cal_maps ? 1 : 0, &st, r.data()),
        "mloam_calib_rig");
  pose_i.t_ = {{pi[0], pi[1], pi[2]}}, pose_i.q_ = {{pi[3], pi[4], pi[5], pi[6]}};  // as solved: PoseLocalParameterization normalised it
  for (size_t n = 0; n < L; n++) {
    const double *x = &ext[7 * n];
    pose_ext[n].t_ = {{x[0], x[1], x[2]}}, pose_ext[n].q_ = {{x[3], x[4], x[5], x[6]}};
  }
  if (rows) *rows = r;
  return st;
}

// ---- pcl::io::loadPCDFile<pcl::PointXYZ> of the dataset nodes (rosNodeRVOxford.cpp:355-370): the file's points as float4 (x, y, z, 0),
// an ASCII body decoded on the device by mloam_pcd_decode.  Returns 0, or -1 when the file cannot be read or is refused, as PCL does.
inline int loadPCDFile(mloam_ctx_t *ctx, const std::string &path, std::vector<mloam_point_t> &cloud) {
  return io::loadPCDPoints(ctx, path, cloud) ? 0 : -1;
}
}  // namespace mloam
