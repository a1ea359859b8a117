// mloam_adapter.hpp — the hot-path classes with the REFERENCE'S OWN types (PCL clouds, Eigen vectors, Ceres bases), for a tree that
// has PCL / Eigen / Ceres: include it INSTEAD of estimator/src/imageSegmenter/image_segmenter.hpp, featureExtract/feature_extract.hpp, lidarTracker/lidar_tracker.h,
// factor/pose_local_parameterization.h and factor/lidar_{map,scan,pure_odom,online_calib}_factor.hpp, AFTER the reference's
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
#include <cstring>
#include <limits>
#include <memory>
#include <stdexcept>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "mloam_context.hpp"

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
    const int method = gf_method == "wo_gf" ? 0 : gf_method == "rnd" ? 1 : gf_method == "fps" ? 2 : 3;  // gd_fix / gd_float
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
};
