// mloam_adapter.hpp — the hot-path classes with the REFERENCE'S OWN types (PCL clouds, Eigen vectors, Ceres bases), for a tree that
// has PCL / Eigen / Ceres: include it INSTEAD of estimator/src/imageSegmenter/image_segmenter.hpp, featureExtract/feature_extract.hpp, lidarTracker/lidar_tracker.h,
// factor/pose_local_parameterization.h, factor/lidar_{map,scan,pure_odom,online_calib}_factor.hpp and factor/prior_factor.hpp, AFTER the reference's
// parameters.h (ScanInfo, cloudFeature, PointPlaneFeature), pose.h (Pose) and <pcl/point_cloud.h>, <Eigen/Dense>, <ceres/ceres.h>.
//
// What keeps compiling unchanged: every call of FeatureExtract::extractCloud / match*FromMap / match*FromScan / match*PointFromMap
// (same template parameter, argument order and defaults as feature_extract.hpp:74-128), LidarTracker::trackCloud and the public
// member f_extract_ (lidar_tracker.h:44-52), PoseLocalParameterization (Plus / ComputeJacobian / GlobalSize / LocalSize /
// setParameter / is_degenerate_ / Eigen V_update_), every factor constructor (Eigen::Vector3d point, Vector4d / VectorXd coeff,
// s | Matrix3d cov | sqrt_info) and Evaluate(), ActiveFeatureSelection::goodFeatureMatching with the argument list of lidar_mapper.h:229.
// What a maintainer edits: the kd-tree VARIABLES change type from pcl::KdTreeFLANN<PointType> to mloam::KdTreeFLANN<PointType> at
// their declarations (lidar_tracker.cpp:27-34, lidar_mapper.h:86-87, estimator.cpp:1122-1123,1229-1232) — same ::Ptr, setInputCloud
// and nearestKSearch members; LidarTracker::evalDegenracy (unused in the reference) is not provided.
//
// tests/stubs/ holds minimal stand-ins for those third-party headers so that this file is compile-checked in CI without them
// (tests/test_abi_cpu.py::test_adapter_compiles_against_stub_headers); with the real headers nothing here changes.
#pragma once
#include <cmath>
#include <cstdio>
#include <cstring>
#include <initializer_list>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "mloam_context.hpp"
#include "mloam_io.hpp"

namespace mloam {

template <typename PointT>
inline std::vector<mloam_point_t> packCloud(const pcl::PointCloud<PointT> &c) {
  std::vector<mloam_point_t> v(c.size());
  for (size_t i = 0; i < c.size(); i++) v[i] = mloam_point_t{c.points[i].x, c.points[i].y, c.points[i].z, c.points[i].intensity};
  return v;
}
inline void unpackCloud(const mloam_point_t *p, int n, common::PointICloud &c) {
  c.clear();
  c.resize((size_t)n);
  for (int i = 0; i < n; i++) c.points[i].x = p[i].x, c.points[i].y = p[i].y, c.points[i].z = p[i].z, c.points[i].intensity = p[i].intensity;
}
inline void poseToParam(const Pose &p, double *x) {  // [tx ty tz qx qy qz qw], pose_local_parameterization.h:20
  x[0] = p.t_(0), x[1] = p.t_(1), x[2] = p.t_(2), x[3] = p.q_.x(), x[4] = p.q_.y(), x[5] = p.q_.z(), x[6] = p.q_.w();
}

// Drop-in for pcl::KdTreeFLANN<PointT>: a map slot of the calling thread's GPU context.  Slots are handed out round-robin among the
// context's MLOAM_NUM_MAPS = 4 (the reference never has more than two trees alive per thread plus the tracker's two).
template <typename PointT>
class KdTreeFLANN {
 public:
  typedef std::shared_ptr<KdTreeFLANN<PointT>> Ptr;
  typedef typename pcl::PointCloud<PointT>::ConstPtr PointCloudConstPtr;
  explicit KdTreeFLANN(int slot = -1) : slot_(slot >= 0 ? slot : nextSlot()) {}
  void setInputCloud(const PointCloudConstPtr &cloud) {
    std::vector<mloam_point_t> v = packCloud(*cloud);
    check(ThreadContext::get(), mloam_map_build(ThreadContext::get(), slot_, v.data(), (int)v.size(), 0.f), "mloam_map_build");
  }
  // exact K nearest like FLANN (no radius limit); k in {1, 5, 10}
  int nearestKSearch(const PointT &p, int k, std::vector<int> &k_indices, std::vector<float> &k_sqr_distances) const {
    k_indices.assign(k, -1);
    k_sqr_distances.assign(k, std::numeric_limits<float>::infinity());
    const mloam_point_t q{p.x, p.y, p.z, p.intensity};
    check(ThreadContext::get(), mloam_knn(ThreadContext::get(), slot_, &q, 1, nullptr, k, 1.0e12f, k_indices.data(), k_sqr_distances.data()), "mloam_knn");
    int got = 0;
    while (got < k && k_indices[got] >= 0) got++;
    k_indices.resize(got), k_sqr_distances.resize(got);
    return got;
  }
  int slot() const { return slot_; }

 private:
  static int nextSlot() {
    thread_local int next = 0;
    const int s = next;
    next = (next + 1) % MLOAM_NUM_MAPS;
    return s;
  }
  int slot_;
};

}  // namespace mloam

// ----------------------------------------------------------------------------------------------- ImageSegmenter
// imageSegmenter/image_segmenter.hpp:47-84.  segmentCloud with scan_info.segment_flag_ == false (`segment_cloud: 0`: projection onto the
// range image, first point of a pixel wins, intensity += ring, ring-ordered output, ScanInfo) runs on the GPU; the BFS labelling of
// `segment_cloud: 1` (image_segmenter.hpp:160-360) is not provided and throws.
extern double ROI_RANGE;  // parameters.h:86
extern float SCAN_PERIOD;  // parameters.h:78
class ImageSegmenter {
 public:
  ImageSegmenter() {}
  void setParameter(const int &vertical_scans, const int &horizon_scans, const int &min_cluster_size, const int &segment_valid_point_num,
                    const int &segment_valid_line_num) {
    vertical_scans_ = vertical_scans, horizon_scans_ = horizon_scans;
    (void)min_cluster_size, (void)segment_valid_point_num, (void)segment_valid_line_num;  // BFS labelling only
  }
  template <typename PointType>
  void segmentCloud(const typename pcl::PointCloud<PointType> &laser_cloud_in, typename pcl::PointCloud<PointType> &laser_cloud_out,
                    typename pcl::PointCloud<PointType> &laser_cloud_outlier, ScanInfo &scan_info) {
    if (scan_info.segment_flag_) throw std::runtime_error("mloam::ImageSegmenter: segment_cloud: 1 (BFS labelling) is not provided");
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> in = mloam::packCloud(laser_cloud_in);
    std::vector<mloam_point_t> out(in.size() + 1);
    int n_out = 0;
    scan_info.scan_start_ind_.resize(vertical_scans_), scan_info.scan_end_ind_.resize(vertical_scans_);
    mloam::check(ctx, mloam_project_cloud(ctx, in.data(), (int)in.size(), vertical_scans_, horizon_scans_, ROI_RANGE, out.data(), &n_out,
                                          scan_info.scan_start_ind_.data(), scan_info.scan_end_ind_.data()), "mloam_project_cloud");
    laser_cloud_out.clear();
    laser_cloud_out.resize((size_t)n_out);
    for (int i = 0; i < n_out; i++) {
      PointType &q = laser_cloud_out.points[i];
      q.x = out[i].x, q.y = out[i].y, q.z = out[i].z, q.intensity = out[i].intensity;
    }
    if (n_out > 0) laser_cloud_outlier.push_back(laser_cloud_out.points[0]);  // image_segmenter.hpp:388
  }

 private:
  int vertical_scans_ = 64, horizon_scans_ = 2048;
};

// ----------------------------------------------------------------------------------------------- FeatureExtract
class FeatureExtract {
 public:
  FeatureExtract() {}

  void extractCloud(const common::PointICloud &laser_cloud_in, const ScanInfo &scan_info, cloudFeature &cloud_feature) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> in = mloam::packCloud(laser_cloud_in);
    const int n = (int)in.size();
    std::vector<mloam_point_t> b0(n + 1), b1(n + 1), b2(n + 1), b3(n + 1);
    mloam_features_t f;
    f.corner_points_sharp = b0.data(), f.corner_points_less_sharp = b1.data(), f.surf_points_flat = b2.data(), f.surf_points_less_flat = b3.data();
    f.cap = n;
    mloam::check(ctx, mloam_extract_features(ctx, in.data(), n, scan_info.scan_start_ind_.data(), scan_info.scan_end_ind_.data(),
                                             (int)scan_info.scan_start_ind_.size(), &f), "mloam_extract_features");
    cloud_feature.clear();
    cloud_feature["laser_cloud"] = laser_cloud_in;  // feature_extract.cpp:281-285
    mloam::unpackCloud(b0.data(), f.n_sharp, cloud_feature["corner_points_sharp"]);
    mloam::unpackCloud(b1.data(), f.n_less_sharp, cloud_feature["corner_points_less_sharp"]);
    mloam::unpackCloud(b2.data(), f.n_flat, cloud_feature["surf_points_flat"]);
    mloam::unpackCloud(b3.data(), f.n_less_flat, cloud_feature["surf_points_less_flat"]);
  }
  void calTimestampPacked(const std::vector<mloam_point_t> &in, int time_field, common::PointICloud &laser_cloud_out) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> out(in.size() + 1);
    int n_out = 0;
    mloam::check(ctx, mloam_cal_timestamp(ctx, in.data(), (int)in.size(), time_field, SCAN_PERIOD, out.data(), &n_out), "mloam_cal_timestamp");
    mloam::unpackCloud(out.data(), n_out, laser_cloud_out);
  }

#ifdef POINTWITHTIME_HPP
  // calTimestamp (feature_extract.hpp:68-72, feature_extract.cpp:38-114) on the GPU, provided where mloam_pcl/point_with_time.hpp is included
  // first (as feature_extract.hpp:42 does).  The reference gets clouds the driver node already passed through removeNaNFromPointCloud;
  // here a point with a non-finite x, y or z is dropped, so both orders give the same cloud.  SCAN_PERIOD: parameters.h:78.
  void calTimestamp(const common::PointCloud &laser_cloud_in, common::PointICloud &laser_cloud_out) {
    std::vector<mloam_point_t> in(laser_cloud_in.size());
    for (size_t i = 0; i < in.size(); i++) in[i] = mloam_point_t{laser_cloud_in.points[i].x, laser_cloud_in.points[i].y, laser_cloud_in.points[i].z, 0.f};
    calTimestampPacked(in, 0, laser_cloud_out);
  }
  void calTimestamp(const common::PointITimeCloud &laser_cloud_in, common::PointICloud &laser_cloud_out) {
    std::vector<mloam_point_t> in(laser_cloud_in.size());  // PointXYZIWithTime::timestamp [us] rides in the w lane
    for (size_t i = 0; i < in.size(); i++)
      in[i] = mloam_point_t{laser_cloud_in.points[i].x, laser_cloud_in.points[i].y, laser_cloud_in.points[i].z, laser_cloud_in.points[i].timestamp};
    calTimestampPacked(in, 1, laser_cloud_out);
  }
#endif

  template <typename PointType>
  void matchCornerFromScan(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_corner_from_scan, const typename pcl::PointCloud<PointType> &cloud_scan,
                           const typename pcl::PointCloud<PointType> &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    matchFromScan<PointType>('c', kdtree_corner_from_scan, cloud_scan, cloud_data, pose_local, features);
  }
  template <typename PointType>
  void matchSurfFromScan(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_surf_from_scan, const typename pcl::PointCloud<PointType> &cloud_scan,
                         const typename pcl::PointCloud<PointType> &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    matchFromScan<PointType>('s', kdtree_surf_from_scan, cloud_scan, cloud_data, pose_local, features);
  }
  template <typename PointType>
  void matchCornerFromMap(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_corner_from_map, const typename pcl::PointCloud<PointType> &cloud_map,
                          const typename pcl::PointCloud<PointType> &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features,
                          const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    matchFromMap<PointType>('c', kdtree_corner_from_map, cloud_map, cloud_data, pose_local, features, N_NEIGH, CHECK_FOV);
  }
  template <typename PointType>
  void matchSurfFromMap(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_surf_from_map, const typename pcl::PointCloud<PointType> &cloud_map,
                        const typename pcl::PointCloud<PointType> &cloud_data, const Pose &pose_local, std::vector<PointPlaneFeature> &features,
                        const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    matchFromMap<PointType>('s', kdtree_surf_from_map, cloud_map, cloud_data, pose_local, features, N_NEIGH, CHECK_FOV);
  }
  template <typename PointType>
  bool matchCornerPointFromMap(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_corner_from_map, const typename pcl::PointCloud<PointType> &cloud_map,
                               const PointType &point_ori, const Pose &pose_local, PointPlaneFeature &feature, const size_t &idx,
                               const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    return matchPointFromMap<PointType>('c', kdtree_corner_from_map, cloud_map, point_ori, pose_local, feature, idx, N_NEIGH, CHECK_FOV);
  }
  template <typename PointType>
  bool matchSurfPointFromMap(const typename mloam::KdTreeFLANN<PointType>::Ptr &kdtree_surf_from_map, const typename pcl::PointCloud<PointType> &cloud_map,
                             const PointType &point_ori, const Pose &pose_local, PointPlaneFeature &feature, const size_t &idx,
                             const size_t &N_NEIGH = 5, const bool &CHECK_FOV = true) {
    return matchPointFromMap<PointType>('s', kdtree_surf_from_map, cloud_map, point_ori, pose_local, feature, idx, N_NEIGH, CHECK_FOV);
  }

 private:
  static void fillFeature(PointPlaneFeature &f, size_t idx, const mloam_point_t &q, const double *coeffs, char type, int n_coeff) {
    f.idx_ = idx;
    f.point_ = Eigen::Vector3d((double)q.x, (double)q.y, (double)q.z);
    f.coeffs_.resize(n_coeff);
    for (int k = 0; k < n_coeff; k++) f.coeffs_(k) = coeffs[k];
    f.laser_idx_ = (size_t)q.intensity;
    f.type_ = type;
  }
  template <typename PointType>
  void matchFromMap(char type, const typename mloam::KdTreeFLANN<PointType>::Ptr &kd, const pcl::PointCloud<PointType> &, const pcl::PointCloud<PointType> &cloud_data,
                    const Pose &pose_local, std::vector<PointPlaneFeature> &features, size_t n_neigh, bool check_fov) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    mloam_params_t &P = mloam::ThreadContext::params();
    P.n_neigh = (int)n_neigh, P.check_fov = check_fov ? 1 : 0;
    mloam::ThreadContext::applyParams();
    std::vector<mloam_point_t> q = mloam::packCloud(cloud_data);
    const int n = (int)q.size();
    std::vector<unsigned char> valid(n + 1);
    std::vector<double> coeffs((size_t)n * 6 + 6);
    double x[7];
    mloam::poseToParam(pose_local, x);
    mloam::check(ctx, mloam_match_from_map(ctx, kd->slot(), type, q.data(), n, x, valid.data(), coeffs.data(), nullptr), "mloam_match_from_map");
    features.clear();  // compacted in query order (feature_extract.hpp:398-399, :536-537)
    for (int i = 0; i < n; i++) {
      if (!valid[i]) continue;
      PointPlaneFeature f;
      fillFeature(f, (size_t)i, q[i], &coeffs[(size_t)i * 6], type, type == 's' ? 4 : 6);
      features.push_back(f);
    }
  }
  template <typename PointType>
  bool matchPointFromMap(char type, const typename mloam::KdTreeFLANN<PointType>::Ptr &kd, const pcl::PointCloud<PointType> &map, const PointType &p,
                         const Pose &pose, PointPlaneFeature &feature, size_t idx, size_t n_neigh, bool check_fov) {
    pcl::PointCloud<PointType> one;
    one.push_back(p);
    std::vector<PointPlaneFeature> fs;
    matchFromMap<PointType>(type, kd, map, one, pose, fs, n_neigh, check_fov);
    if (fs.empty()) return false;
    feature = fs[0];
    feature.idx_ = idx;
    return true;
  }
  template <typename PointType>
  void matchFromScan(char type, const typename mloam::KdTreeFLANN<PointType>::Ptr &kd, const pcl::PointCloud<PointType> &, const pcl::PointCloud<PointType> &cloud_data,
                     const Pose &pose_local, std::vector<PointPlaneFeature> &features) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> q = mloam::packCloud(cloud_data);
    const int n = (int)q.size();
    std::vector<unsigned char> valid(n + 1);
    std::vector<double> coeffs((size_t)n * 6 + 6);
    double x[7];
    mloam::poseToParam(pose_local, x);
    mloam::check(ctx, mloam_match_from_scan(ctx, kd->slot(), type, q.data(), n, x, valid.data(), coeffs.data(), nullptr), "mloam_match_from_scan");
    features.clear();
    for (int i = 0; i < n; i++) {
      if (!valid[i]) continue;
      PointPlaneFeature f;
      fillFeature(f, (size_t)i, q[i], &coeffs[(size_t)i * 6], type == 's' ? 's' : 'n', type == 's' ? 4 : 6);  // scan corners keep type_ 'n' (:262-266)
      f.laser_idx_ = 0;
      features.push_back(f);
    }
  }
};

// ----------------------------------------------------------------------------------------------- parameterisation
class PoseLocalParameterization : public ceres::LocalParameterization {
  virtual bool Plus(const double *x, const double *delta, double *x_plus_delta) const {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    double V[36];
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) V[i * 6 + j] = V_update_(i, j);  // row-major for the ABI whatever Eigen's storage order is
    mloam::check(ctx, mloam_pose_plus(ctx, x, delta, V, x_plus_delta), "mloam_pose_plus");
    return true;
  }
  virtual bool ComputeJacobian(const double *, double *jacobian) const {  // 7x6 row-major [I6; 0] (pose_local_parameterization.cpp:50-56)
    for (int i = 0; i < 42; i++) jacobian[i] = 0.0;
    for (int i = 0; i < 6; i++) jacobian[i * 6 + i] = 1.0;
    return true;
  }
  virtual int GlobalSize() const { return 7; }
  virtual int LocalSize() const { return 6; }

 public:
  PoseLocalParameterization() { setParameter(); }
  void setParameter() {
    is_degenerate_ = false;
    V_update_ = Eigen::Matrix<double, 6, 6>::Identity();
  }
  bool is_degenerate_;
  Eigen::Matrix<double, 6, 6> V_update_;
};

// ----------------------------------------------------------------------------------------------- factors
namespace mloam {
// One factor = a batch of one through mloam_factor_evaluate; ROWS x (7 per block) Jacobians, row-major, last column zero.
template <int ROWS, int BLOCKS>
class FactorImpl {
 protected:
  FactorImpl(int kind, const Eigen::Vector3d &point, const double *coeff, int n_coeff, double sqrt_info) : kind_(kind), sqrt_info_(sqrt_info) {
    for (int k = 0; k < 3; k++) point_[k] = point(k);
    for (int k = 0; k < 6; k++) coeff_[k] = k < n_coeff ? coeff[k] : 0.0;
  }
  bool evaluate(double const *const *param, double *residuals, double **jacobians) const {
    mloam_ctx_t *ctx = ThreadContext::get();
    double x[21];
    for (int b = 0; b < BLOCKS; b++) std::memcpy(x + 7 * b, param[b], 7 * sizeof(double));
    double J[63];
    check(ctx, mloam_factor_evaluate(ctx, kind_, 1, point_, coeff_, &sqrt_info_, x, residuals, jacobians ? J : nullptr), "mloam_factor_evaluate");
    if (jacobians) {  // null-tolerant on each block, as Ceres requires
      if (BLOCKS == 1) {
        if (jacobians[0]) std::memcpy(jacobians[0], J, sizeof(double) * ROWS * 7);
      } else {
        for (int b = 0; b < BLOCKS; b++)
          if (jacobians[b]) std::memcpy(jacobians[b], J + 7 * b, sizeof(double) * 7);
      }
    }
    return true;
  }
  int kind_;
  double point_[3], coeff_[6], sqrt_info_;
};
inline double mapSqrtInfo(const Eigen::Matrix3d &cov_matrix) {  // lidar_map_factor.hpp:34,41
  const double s = std::sqrt(1 / cov_matrix.trace());
  return s >= 3.0 ? 1.0 : s / 3.0;
}
}  // namespace mloam

#define MLOAM_FACTOR(NAME, ROWS, BLOCKS, KIND, COEFF_T, NCOEF, THIRD_T, THIRD_DEFAULT, SQRT_INFO_EXPR)                                      \
  class NAME : public ceres::SizedCostFunction<ROWS, 7>, private mloam::FactorImpl<ROWS, BLOCKS> {                                          \
   public:                                                                                                                                  \
    NAME(const Eigen::Vector3d &point, const COEFF_T &coeff, const THIRD_T &third = THIRD_DEFAULT)                                           \
        : mloam::FactorImpl<ROWS, BLOCKS>(KIND, point, coeff.data(), NCOEF, SQRT_INFO_EXPR) {}                                               \
    bool Evaluate(double const *const *param, double *residuals, double **jacobians) const { return this->evaluate(param, residuals, jacobians); } \
  }
// lidar_map_factor.hpp:26-126 / :130-235 (cov_matrix -> clamped sqrt_info)
MLOAM_FACTOR(LidarMapPlaneNormFactor, 1, 1, 0, Eigen::Vector4d, 4, Eigen::Matrix3d, Eigen::Matrix3d::Identity(), mloam::mapSqrtInfo(third));
MLOAM_FACTOR(LidarMapEdgeFactor, 1, 1, 1, Eigen::VectorXd, 6, Eigen::Matrix3d, Eigen::Matrix3d::Identity(), mloam::mapSqrtInfo(third));
// lidar_scan_factor.hpp:25-126 / :130-232 / :236-343 (s = 1: the distortion slerp is the identity)
MLOAM_FACTOR(LidarScanPlaneNormFactor, 1, 1, 0, Eigen::Vector4d, 4, double, 1.0, ((void)third, 1.0));
MLOAM_FACTOR(LidarScanEdgeFactor, 1, 1, 1, Eigen::VectorXd, 6, double, 1.0, ((void)third, 1.0));
MLOAM_FACTOR(LidarScanEdgeFactorVector, 3, 1, 2, Eigen::VectorXd, 6, double, 1.0, ((void)third, 1.0));
// lidar_online_calib_factor.hpp:24-121 / :125-227
MLOAM_FACTOR(LidarOnlineCalibPlaneNormFactor, 1, 1, 0, Eigen::Vector4d, 4, double, 1.0, third);
MLOAM_FACTOR(LidarOnlineCalibEdgeFactor, 1, 1, 1, Eigen::VectorXd, 6, double, 1.0, third);
#undef MLOAM_FACTOR
// lidar_pure_odom_factor.hpp:27-195 / :198-381 — parameter blocks (pivot, pose_i, ext): SizedCostFunction<1, 7, 7, 7>
#define MLOAM_ODOM_FACTOR(NAME, KIND, COEFF_T, NCOEF)                                                                                      \
  class NAME : public ceres::SizedCostFunction<1, 7, 7, 7>, private mloam::FactorImpl<1, 3> {                                             \
   public:                                                                                                                                \
    NAME(const Eigen::Vector3d &point, const COEFF_T &coeff, const double &sqrt_info = 1.0)                                                \
        : mloam::FactorImpl<1, 3>(KIND, point, coeff.data(), NCOEF, sqrt_info) {}                                                          \
    bool Evaluate(double const *const *param, double *residuals, double **jacobians) const { return this->evaluate(param, residuals, jacobians); } \
  }
MLOAM_ODOM_FACTOR(LidarPureOdomPlaneNormFactor, 3, Eigen::Vector4d, 4);
MLOAM_ODOM_FACTOR(LidarPureOdomEdgeFactor, 4, Eigen::VectorXd, 6);
#undef MLOAM_ODOM_FACTOR
// prior_factor.hpp:27-72 — PriorFactor(pos, rot, pos_scale, rot_scale) on one pose block, evaluated on the host (6 residuals):
// residual = diag(pos_scale I3, rot_scale I3) [P - pos ; 2 (rot^-1 Q).vec], jacobian = the same scales times diag(I3,
// LeftQuatMatrix(Q^-1 rot).topLeftCorner<3,3>()) with a zero 7th column — as the reference writes it (its comment: "seem to be
// wrong"), so that a problem built with it is the one the reference solves.  Eigen's inverse() is conjugate / squaredNorm.  The same
// statement is what mloam_calib_rig adds on the device.
class PriorFactor : public ceres::SizedCostFunction<6, 7> {
 public:
  PriorFactor(const Eigen::Vector3d &pos, const Eigen::Quaterniond &rot, const double &pos_scale, const double &rot_scale)
      : pos_scale_(pos_scale), rot_scale_(rot_scale) {
    x0_[0] = pos(0), x0_[1] = pos(1), x0_[2] = pos(2), x0_[3] = rot.x(), x0_[4] = rot.y(), x0_[5] = rot.z(), x0_[6] = rot.w();
  }
  bool Evaluate(double const *const *param, double *residuals, double **jacobians) const {
    const double *x = param[0];
    const double q[4] = {x[3], x[4], x[5], x[6]}, r0[4] = {x0_[3], x0_[4], x0_[5], x0_[6]};
    double qi[4], e[4];
    inv(r0, qi), mul(qi, q, e);
    for (int k = 0; k < 3; k++) residuals[k] = pos_scale_ * (x[k] - x0_[k]), residuals[3 + k] = rot_scale_ * (2 * e[k]);
    if (jacobians && jacobians[0]) {
      double m[4];
      inv(q, qi), mul(qi, r0, m);
      const double L[9] = {m[3], -m[2], m[1], m[2], m[3], -m[0], -m[1], m[0], m[3]};  // w I + [v]x
      double *J = jacobians[0];
      for (int k = 0; k < 42; k++) J[k] = 0.0;
      for (int k = 0; k < 3; k++) J[k * 7 + k] = pos_scale_;
      for (int i = 0; i < 3; i++)
        for (int j = 0; j < 3; j++) J[(3 + i) * 7 + 3 + j] = rot_scale_ * L[i * 3 + j];
    }
    return true;
  }

 private:
  static void inv(const double *q, double *o) {  // [x y z w]
    const double n2 = q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3];
    o[0] = -q[0] / n2, o[1] = -q[1] / n2, o[2] = -q[2] / n2, o[3] = q[3] / n2;
  }
  static void mul(const double *a, const double *b, double *o) {
    o[0] = a[3] * b[0] + a[0] * b[3] + a[1] * b[2] - a[2] * b[1], o[1] = a[3] * b[1] + a[1] * b[3] + a[2] * b[0] - a[0] * b[2];
    o[2] = a[3] * b[2] + a[2] * b[3] + a[0] * b[1] - a[1] * b[0], o[3] = a[3] * b[3] - a[0] * b[0] - a[1] * b[1] - a[2] * b[2];
  }
  double x0_[7], pos_scale_, rot_scale_;
};

// ----------------------------------------------------------------------------------------------- LidarTracker
class LidarTracker {
 public:
  LidarTracker() {}
  Pose trackCloud(const cloudFeature &prev_cloud_feature, const cloudFeature &cur_cloud_feature, const Pose &pose_ini) {
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> a = mloam::packCloud(prev_cloud_feature.find("corner_points_less_sharp")->second);
    std::vector<mloam_point_t> b = mloam::packCloud(prev_cloud_feature.find("surf_points_less_flat")->second);
    std::vector<mloam_point_t> c = mloam::packCloud(cur_cloud_feature.find("corner_points_sharp")->second);
    std::vector<mloam_point_t> d = mloam::packCloud(cur_cloud_feature.find("surf_points_flat")->second);
    double x[7], y[7];
    mloam::poseToParam(pose_ini, x);
    mloam::check(ctx, mloam_track_cloud(ctx, a.data(), (int)a.size(), b.data(), (int)b.size(), c.data(), (int)c.size(), d.data(), (int)d.size(), x, y, nullptr),
                 "mloam_track_cloud");
    return Pose(Eigen::Quaterniond(y[6], y[3], y[4], y[5]), Eigen::Vector3d(y[0], y[1], y[2]));  // lidar_tracker.cpp:126-128
  }
  FeatureExtract f_extract_;
};

// ----------------------------------------------------------------------------------------------- good features (mapper)
// ActiveFeatureSelection::goodFeatureMatching with the reference's argument list (lidar_mapper.h:229-238).  `seed` replaces
// std::random_device; the wall-clock cap is dropped (see include/mloam_b200.h).
class ActiveFeatureSelection {
 public:
  unsigned long long seed = 0;
  void goodFeatureMatching(const mloam::KdTreeFLANN<common::PointIWithCov>::Ptr &kdtree_from_map, const common::PointICovCloud &laser_map,
                           const common::PointICovCloud &laser_cloud, const Pose &pose_local, std::vector<PointPlaneFeature> &all_features,
                           std::vector<size_t> &sel_feature_idx, const char feature_type, const std::string gf_method, const double gf_ratio,
                           Eigen::Matrix<double, 6, 6> &sub_mat_H) {
    (void)laser_map;
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    // gd_fix / gd_float are one selection; gd_float's ratio policy (lidar_mapper_keyframe.cpp:456-495) is mloam_set_gf_float
    const int method = gf_method == "wo_gf" ? 0 : gf_method == "rnd" ? 1 : gf_method == "fps" ? 2 : 3;
    std::vector<mloam_point_t> pts = mloam::packCloud(laser_cloud);
    const int n = (int)pts.size();
    std::vector<float> cov6((size_t)n * 6 + 6);
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 6; k++) cov6[(size_t)i * 6 + k] = laser_cloud.points[i].cov_vec[k];
    std::vector<int> sel(n + 1);
    std::vector<unsigned char> matched(n + 1), valid(n + 1);
    std::vector<double> jaco((size_t)n * 6 + 6), coeffs((size_t)n * 6 + 6);
    int n_sel = 0;
    double x[7], H[36];
    mloam::poseToParam(pose_local, x);
    mloam_params_t &P = mloam::ThreadContext::params();
    P.n_neigh = 5, P.check_fov = 0;  // lidar_mapper.h:253, :193-283
    mloam::ThreadContext::applyParams();
    mloam::check(ctx, mloam_good_features(ctx, kdtree_from_map->slot(), feature_type, pts.data(), n, cov6.data(), x, method, gf_ratio, seed++, sel.data(),
                                          &n_sel, H, matched.data(), jaco.data()), "mloam_good_features");
    mloam::check(ctx, mloam_match_from_map(ctx, kdtree_from_map->slot(), feature_type, pts.data(), n, x, valid.data(), coeffs.data(), nullptr),
                 "mloam_match_from_map");
    all_features.assign((size_t)n, PointPlaneFeature());  // :240-241, filled for the matched ones
    for (int i = 0; i < n; i++) {
      if (!matched[i]) continue;
      PointPlaneFeature &f = all_features[i];
      f.idx_ = (size_t)i, f.laser_idx_ = (size_t)pts[i].intensity, f.type_ = feature_type;
      f.point_ = Eigen::Vector3d((double)pts[i].x, (double)pts[i].y, (double)pts[i].z);
      const int nc = feature_type == 's' ? 4 : 6;
      f.coeffs_.resize(nc);
      for (int k = 0; k < nc; k++) f.coeffs_(k) = coeffs[(size_t)i * 6 + k];
      f.jaco_.resize(1, 6);
      for (int k = 0; k < 6; k++) f.jaco_(0, k) = jaco[(size_t)i * 6 + k];
    }
    sel_feature_idx.assign(sel.begin(), sel.begin() + n_sel);
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) sub_mat_H(i, j) = H[i * 6 + j];
  }
  // ActiveFeatureSelection::evalFullHessian with the reference's argument list (lidar_mapper.h:176-182): mat_H and feat_num accumulate
  void evalFullHessian(const mloam::KdTreeFLANN<common::PointIWithCov>::Ptr &kdtree_from_map, const common::PointICovCloud &laser_map,
                       const common::PointICovCloud &laser_cloud, const Pose &pose_local, const char feature_type,
                       Eigen::Matrix<double, 6, 6> &mat_H, int &feat_num) {
    (void)laser_map;
    mloam_ctx_t *ctx = mloam::ThreadContext::get();
    std::vector<mloam_point_t> pts = mloam::packCloud(laser_cloud);
    const int n = (int)pts.size();
    std::vector<float> cov6((size_t)n * 6 + 6);
    for (int i = 0; i < n; i++)
      for (int k = 0; k < 6; k++) cov6[(size_t)i * 6 + k] = laser_cloud.points[i].cov_vec[k];
    double x[7], H[36];
    mloam::poseToParam(pose_local, x);
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) H[i * 6 + j] = mat_H(i, j);
    mloam::check(ctx, mloam_full_hessian(ctx, kdtree_from_map->slot(), feature_type, pts.data(), n, cov6.data(), x, H, &feat_num), "mloam_full_hessian");
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) mat_H(i, j) = H[i * 6 + j];
  }
};

// ---- DISTORTION (estimator.cpp:545-590).  Estimator::process computes pose_undist and calls undistortMeasurements(pose_undist) on the
// features the mapper takes; with the frame on the device those features are moved inside the next mloam_frame* call of ctx, the context
// that runs the frames:
//   mloam::setDistortion(ctx, DISTORTION, SCAN_PERIOD);                                    once, after mloam_set_lidars
//   pose_undist = mloam::undistortPoses(pose_rlt_[IDX_REF], qbl_, tbl_);                    estimator.cpp:575-579
//   mloam::undistortMeasurements(ctx, pose_undist, IDX_REF, ESTIMATE_EXTRINSIC);           in place of Estimator::undistortMeasurements
// or, when the odometry has sweep k+1's pose_undist before the mapper takes it (the node split: the odometry undistorts sweep k+1 while
// the mapper solves sweep k), with that sweep's announcement:
//   mloam_frame_set_next(ctx, ...sweep k+1...);
//   mloam::undistortMeasurementsNext(ctx, pose_undist_next, IDX_REF, ESTIMATE_EXTRINSIC);  the look-ahead undistorts it too
namespace mloam {
inline void setDistortion(mloam_ctx_t *ctx, bool on, float scan_period) {
  check(ctx, mloam_set_distortion(ctx, on ? 1 : 0, scan_period), "mloam_set_distortion");
}
// pose_undist[n] = Pose(qbl[n], tbl[n]).inverse() * pose_rlt * Pose(qbl[n], tbl[n]) for every LiDAR n; pose_rlt as the Pose holds it
inline std::vector<Pose> undistortPoses(const Pose &pose_rlt, const std::vector<Eigen::Quaterniond> &qbl, const std::vector<Eigen::Vector3d> &tbl) {
  const size_t n = qbl.size();
  std::vector<double> e(7 * n), out(7 * n);
  for (size_t l = 0; l < n; l++) {
    double *x = &e[7 * l];
    x[0] = tbl[l](0), x[1] = tbl[l](1), x[2] = tbl[l](2), x[3] = qbl[l].x(), x[4] = qbl[l].y(), x[5] = qbl[l].z(), x[6] = qbl[l].w();
  }
  double r[7];
  poseToParam(pose_rlt, r);
  if (n == 0 || mloam_undistort_poses(r, 0, (int)n, e.data(), 2, out.data()) != MLOAM_OK)  // 2: every LiDAR its own
    throw std::runtime_error("mloam_undistort_poses: 1..16 LiDARs");
  std::vector<Pose> res(n);
  for (size_t l = 0; l < n; l++) {
    const double *o = &out[7 * l];
    res[l].q_ = Eigen::Quaterniond(o[6], o[3], o[4], o[5]), res[l].t_ = Eigen::Vector3d(o[0], o[1], o[2]);  // normalised already
  }
  return res;
}
// undistortMeasurements (:376-408): LiDAR n's features move with pose_undist[n] when estimate_extrinsic == 2, else with
// pose_undist[idx_ref]; the poses go to the next mloam_frame* call of ctx
inline void undistortMeasurements(mloam_ctx_t *ctx, const std::vector<Pose> &pose_undist, size_t idx_ref, int estimate_extrinsic) {
  std::vector<double> x(7 * pose_undist.size());
  for (size_t l = 0; l < pose_undist.size(); l++) poseToParam(pose_undist[estimate_extrinsic == 2 ? l : idx_ref], &x[7 * l]);
  check(ctx, mloam_frame_undistort(ctx, (int)pose_undist.size(), x.data()), "mloam_frame_undistort");
}
// the same poses for the sweep announced by the last mloam_frame_set_next* call of ctx: the call that takes that sweep needs no
// undistortMeasurements
inline void undistortMeasurementsNext(mloam_ctx_t *ctx, const std::vector<Pose> &pose_undist, size_t idx_ref, int estimate_extrinsic) {
  std::vector<double> x(7 * pose_undist.size());
  for (size_t l = 0; l < pose_undist.size(); l++) poseToParam(pose_undist[estimate_extrinsic == 2 ? l : idx_ref], &x[7 * l]);
  check(ctx, mloam_frame_set_next_undistort(ctx, (int)pose_undist.size(), x.data()), "mloam_frame_set_next_undistort");
}
}  // namespace mloam

// ---- pubPointCloud (lidar_mapper_keyframe.cpp:690-714): the registered clouds of the last mloam_frame* call of ctx, in the world frame
//   mloam::setRegistered(ctx, true);                                                           once
//   mloam::frameRegistered(ctx, laser_cloud_full_res, laser_cloud_surf_last, laser_cloud_corner_last);    after each mloam_frame*
// in place of the three pointAssociateToMap loops; toROSMsg and publish stay the caller's.
namespace mloam {
inline void setRegistered(mloam_ctx_t *ctx, bool on) { check(ctx, mloam_set_registered(ctx, on ? 1 : 0), "mloam_set_registered"); }
inline void frameRegistered(mloam_ctx_t *ctx, int which, common::PointICloud &out) {
  int n = 0;
  check(ctx, mloam_frame_registered(ctx, which, nullptr, 0, &n), "mloam_frame_registered");
  std::vector<mloam_point_t> pts((size_t)n);
  check(ctx, mloam_frame_registered(ctx, which, pts.data(), n, &n), "mloam_frame_registered");
  unpackCloud(pts.data(), n, out);
}
inline void frameRegistered(mloam_ctx_t *ctx, common::PointICloud &full_res, common::PointICloud &surf_last, common::PointICloud &corner_last) {
  frameRegistered(ctx, MLOAM_REGISTERED_FULL_RES, full_res);
  frameRegistered(ctx, MLOAM_REGISTERED_SURF, surf_last);
  frameRegistered(ctx, MLOAM_REGISTERED_CORNER, corner_last);
}
}  // namespace mloam

// ---- pcl::toROSMsg of the published clouds (pubPointCloud :690-714, pubGlobalMap :780-851), packed on the device by one launch:
//   mloam::toROSMsg(ctx, {MLOAM_MSG_FULL_RES, MLOAM_MSG_SURF_LAST, MLOAM_MSG_CORNER_LAST},
//                   {&laser_cloud_full_res_msg, &laser_cloud_surf_last_msg, &laser_cloud_corner_last_msg});
//   mloam::toROSMsg(ctx, MLOAM_MSG_GLOBAL_MAP0, laser_cloud_map_msg);
// in place of the pointAssociateToMap loops and pcl::toROSMsg; setting header.stamp / frame_id and publishing stay the caller's.  Each
// message's data buffer is reused, so publishers that keep their messages pay one launch a call.  A template on the message type
// (sensor_msgs::PointCloud2), so that this header still compiles in a tree without ROS.
namespace mloam {
template <typename PointCloud2>
inline void toROSMsg(mloam_ctx_t *ctx, const std::vector<int> &sources, std::initializer_list<PointCloud2 *> msgs) {
  const std::vector<PointCloud2 *> out(msgs);
  if (out.size() != sources.size()) throw std::invalid_argument("toROSMsg: one message per source");
  std::vector<std::vector<uint8_t> *> data;
  for (PointCloud2 *m : out) data.push_back(&m->data);
  std::vector<int> width;
  check(ctx, io::cloudMsgs(ctx, sources, data, width), "mloam_cloud_msgs");
  for (size_t k = 0; k < out.size(); k++) {
    const io::PointCloud2View v = io::cloudMsgView(sources[k], (size_t)width[k], data[k]->data());
    PointCloud2 &m = *out[k];
    m.height = v.height, m.width = v.width, m.is_bigendian = v.is_bigendian, m.point_step = v.point_step, m.row_step = v.row_step;
    m.is_dense = v.is_dense;
    m.fields.resize(v.fields.size());
    for (size_t f = 0; f < v.fields.size(); f++)
      m.fields[f].name = v.fields[f].name, m.fields[f].offset = v.fields[f].offset, m.fields[f].datatype = v.fields[f].datatype,
      m.fields[f].count = v.fields[f].count;
  }
}
template <typename PointCloud2>
inline void toROSMsg(mloam_ctx_t *ctx, int source, PointCloud2 &msg) {
  toROSMsg(ctx, {source}, {&msg});
}
}  // namespace mloam

// ---- Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 over the whole rig (estimator.cpp:633-642, 670-787): one call in place of the
// problem assembly (PriorFactor on every extrinsic when PRIOR_FACTOR, LidarPureOdom* of IDX_REF's frame-i features on pose_i,
// LidarOnlineCalib* of every other LiDAR's features on its extrinsic) and ceres::Solve:
//   mloam::calibRig(ctx, IDX_REF, surf, corner, pose_pivot, pose_i, pose_ext, PRIOR_FACTOR ? &pose_ext : nullptr, PRIOR_FACTOR_POS,
//                   PRIOR_FACTOR_ROT, max_outer, NUM_ITERATIONS);
// surf[n] / corner[n]: LiDAR n's features in its sensor frame (frame i for IDX_REF, the pivot or the accumulation for the others).
// pose_i and pose_ext (one Pose per LiDAR, pose_ext[IDX_REF] constant) are in/out; prior: the PriorFactor targets (tbl_ / qbl_), copied
// before the call, so the extrinsics themselves may be passed.  rows (nullable): each LiDAR's feature rows of the last evaluation.
namespace mloam {
inline mloam_solve_stats_t calibRig(mloam_ctx_t *ctx, size_t idx_ref, const std::vector<common::PointICloud> &surf,
                                    const std::vector<common::PointICloud> &corner, const Pose &pose_pivot, Pose &pose_i, std::vector<Pose> &pose_ext,
                                    const std::vector<Pose> *prior, double prior_pos, double prior_rot, int max_outer, int max_inner,
                                    bool own_cal_maps = false, std::vector<int> *rows = nullptr, double huber_a = 1.0) {
  const size_t L = pose_ext.size();
  if (surf.size() != L || corner.size() != L || (prior && prior->size() != L)) throw std::invalid_argument("calibRig: one cloud / prior per LiDAR");
  std::vector<mloam_point_t> s, c;
  std::vector<int> ns(L), nc(L), r(L);
  for (size_t n = 0; n < L; n++) {
    const std::vector<mloam_point_t> a = packCloud(surf[n]), b = packCloud(corner[n]);
    s.insert(s.end(), a.begin(), a.end()), c.insert(c.end(), b.begin(), b.end());
    ns[n] = (int)a.size(), nc[n] = (int)b.size();
  }
  std::vector<double> ext(7 * L), pr(prior ? 7 * L : 0);
  for (size_t n = 0; n < L; n++) {
    poseToParam(pose_ext[n], &ext[7 * n]);
    if (prior) poseToParam((*prior)[n], &pr[7 * n]);
  }
  double pv[7], pi[7];
  poseToParam(pose_pivot, pv), poseToParam(pose_i, pi);
  mloam_solve_stats_t st;
  check(ctx, mloam_calib_rig(ctx, (int)L, (int)idx_ref, s.data(), ns.data(), c.data(), nc.data(), pv, pi, ext.data(), prior ? pr.data() : nullptr,
                             prior ? prior_pos : 0.0, prior ? prior_rot : 0.0, max_outer, max_inner, huber_a, own_cal_maps ? 1 : 0, &st, r.data()),
        "mloam_calib_rig");
  pose_i.q_ = Eigen::Quaterniond(pi[6], pi[3], pi[4], pi[5]), pose_i.t_ = Eigen::Vector3d(pi[0], pi[1], pi[2]);
  for (size_t n = 0; n < L; n++) {
    const double *x = &ext[7 * n];
    pose_ext[n].q_ = Eigen::Quaterniond(x[6], x[3], x[4], x[5]), pose_ext[n].t_ = Eigen::Vector3d(x[0], x[1], x[2]);
  }
  if (rows) *rows = r;
  return st;
}

// ---- pcl::io::loadPCDFile<PointT> (pcl::PointXYZ) of the dataset nodes (rosNodeRVOxford.cpp:355-370, rosNodeRVHercules.cpp:354-368): the file's
// header read on the host (io::resolvePCDHeader), an ASCII body decoded on the device (mloam_pcd_decode: PCL's values bit for bit, the
// bodies PCL would misread refused), a binary one copied.  Returns 0, or -1 when the file cannot be read or is refused, as PCL does.
template <typename PointT>
int loadPCDFile(mloam_ctx_t *ctx, const std::string &path, pcl::PointCloud<PointT> &cloud) {
  std::vector<mloam_point_t> pts;
  if (!io::loadPCDPoints(ctx, path, pts)) return -1;
  cloud.resize(pts.size());
  for (size_t i = 0; i < pts.size(); i++) cloud[i].x = pts[i].x, cloud[i].y = pts[i].y, cloud[i].z = pts[i].z;
  return 0;
}

// ---- pcl::io::savePCDFileASCII / pcl::PCDWriter::write (= writeASCII at precision 8) of pcl::PointXYZ, pcl::PointXYZI and
// pcl::PointXYZIWithCov clouds: the file written on the device by mloam_pcd_encode (the format: include/mloam_b200.h) and saved at path.
// Returns 0, or -1 where PCL fails: an empty cloud (PCL throws IOException and writes nothing) or a file that cannot be written.
namespace detail {
// the point type's fields: cov_vec and cov_trace (PointXYZIWithCov), intensity (PointXYZI), neither (PointXYZ)
template <typename P>
auto pcd_point(const P &p, mloam_point_t &q, float *cov6, float *trace, int) -> decltype(p.cov_vec[0], p.cov_trace, int()) {
  q.intensity = p.intensity;
  for (int k = 0; k < 6; k++) cov6[k] = p.cov_vec[k];
  *trace = p.cov_trace;
  return MLOAM_PCD_XYZI_COV;
}
template <typename P>
auto pcd_point(const P &p, mloam_point_t &q, float *, float *, long) -> decltype(p.intensity, int()) {
  q.intensity = p.intensity;
  return MLOAM_PCD_XYZI;
}
template <typename P>
int pcd_point(const P &, mloam_point_t &, float *, float *, ...) {
  return MLOAM_PCD_XYZ;
}
}  // namespace detail

template <typename PointT>
int savePCDFileASCII(mloam_ctx_t *ctx, const std::string &path, const pcl::PointCloud<PointT> &cloud) {
  const size_t n = cloud.size();
  if (n == 0) return -1;
  std::vector<mloam_point_t> pts(n);
  std::vector<float> cov6(6 * n), trace(n);
  int layout = MLOAM_PCD_XYZ;
  for (size_t i = 0; i < n; i++) {
    pts[i] = mloam_point_t{cloud[i].x, cloud[i].y, cloud[i].z, 0.f};
    layout = detail::pcd_point(cloud[i], pts[i], &cov6[6 * i], &trace[i], 0);
  }
  const mloam_pcd_cloud_t q = {pts.data(), cov6.data(), trace.data(), (int)n, layout};
  std::vector<uint8_t> bytes(384 + n * 15 * (size_t)io::pcdFields(layout));  // the bound the library refuses beyond: one call
  void *dst = bytes.data();
  const size_t cap = bytes.size();
  size_t nb = 0;
  check(ctx, mloam_pcd_encode(ctx, 1, &q, &dst, &cap, &nb), "mloam_pcd_encode");
  bytes.resize(nb);
  return io::savePCD(path, bytes) ? 0 : -1;
}

class PCDWriter {
 public:
  explicit PCDWriter(mloam_ctx_t *ctx) : ctx_(ctx) {}
  template <typename PointT>
  int write(const std::string &path, const pcl::PointCloud<PointT> &cloud) {
    return savePCDFileASCII(ctx_, path, cloud);
  }

 private:
  mloam_ctx_t *ctx_;
};

// saveGlobalMap (lidar_mapper_keyframe.cpp:853-919) from the keyframe store: mloam_global_map(SAVE, kf_leaf 10 m, leaf 2 x MAP_SURF_RES),
// then the three files pcd_writer.write gives, under dir (the reference's "/tmp/"): mloam_mapping_keyframes.pcd (pose_keyframes_3d),
// mloam_mapping_surf_cloud[_wo_ua].pcd and mloam_mapping_corner_cloud[_wo_ua].pcd (maps 0 and 1), written by one launch.  As in the
// reference, a file that PCL would refuse (an empty cloud) ends the save: -1, and the later files are not written.  Returns 0 or -1.
inline int saveGlobalMap(mloam_ctx_t *ctx, const std::string &dir, bool with_ua, float map_surf_res) {
  check(ctx, mloam_global_map(ctx, MLOAM_GLOBAL_MAP_SAVE, nullptr, 0.0, 10.0, 2.f * map_surf_res, nullptr, nullptr, nullptr), "mloam_global_map");
  std::vector<uint8_t> files[3];
  std::vector<std::vector<uint8_t> *> data = {&files[0], &files[1], &files[2]};
  check(ctx, io::cloudPCD(ctx, {MLOAM_PCD_KEYFRAMES, MLOAM_MSG_GLOBAL_MAP0, MLOAM_MSG_GLOBAL_MAP1}, data), "mloam_cloud_pcd");
  const std::string sfx = with_ua ? ".pcd" : "_wo_ua.pcd";
  const std::string names[3] = {"mloam_mapping_keyframes.pcd", "mloam_mapping_surf_cloud" + sfx, "mloam_mapping_corner_cloud" + sfx};
  for (int k = 0; k < 3; k++)
    if (files[k].empty() || !io::savePCD(dir + names[k], files[k])) return -1;
  return 0;
}
}  // namespace mloam
