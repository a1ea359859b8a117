// Compile check of m-loam_b200/host/mloam_adapter.hpp against the stub third-party headers in this directory: instantiates every class
// and template with the reference's call shapes (lidar_tracker.cpp:27-99, lidar_mapper.h:193-283, estimator.cpp:696-779,1135-1149).
// It is compiled and linked (against libmloam_b200.so), never run: the calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_use_everything() {
  FeatureExtract f_extract;
  PointICloud cloud, map;
  ScanInfo scan_info(64, false);
  {  // estimator.cpp:117-122
    ImageSegmenter img_segment;
    img_segment.setParameter(64, 2048, 5, 5, 3);
    PointICloud laser_cloud_segment, laser_cloud_outlier;
    img_segment.segmentCloud<PointI>(cloud, laser_cloud_segment, laser_cloud_outlier, scan_info);
  }
  cloudFeature feat;
  f_extract.extractCloud(cloud, scan_info, feat);

  mloam::KdTreeFLANN<PointI>::Ptr kdtree(new mloam::KdTreeFLANN<PointI>());
  PointICloud::Ptr map_ptr(new PointICloud());
  kdtree->setInputCloud(map_ptr);
  std::vector<int> idx;
  std::vector<float> sqd;
  kdtree->nearestKSearch(PointI(), 5, idx, sqd);

  Pose pose_local;
  std::vector<PointPlaneFeature> features;
  f_extract.matchCornerFromScan<PointI>(kdtree, map, cloud, pose_local, features);
  f_extract.matchSurfFromScan<PointI>(kdtree, map, cloud, pose_local, features);
  f_extract.matchCornerFromMap<PointI>(kdtree, map, cloud, pose_local, features, 10, true);
  f_extract.matchSurfFromMap<PointI>(kdtree, map, cloud, pose_local, features);
  PointPlaneFeature one;
  f_extract.matchCornerPointFromMap<PointI>(kdtree, map, PointI(), pose_local, one, 3, 5, false);
  // the mapper matches PointIWithCov clouds (lidar_mapper.h:193-210)
  mloam::KdTreeFLANN<PointIWithCov>::Ptr kd_cov(new mloam::KdTreeFLANN<PointIWithCov>());
  PointICovCloud cov_map, cov_scan;
  f_extract.matchSurfPointFromMap<PointIWithCov>(kd_cov, cov_map, PointIWithCov(), pose_local, one, 7, 5, false);

  PoseLocalParameterization *lp = new PoseLocalParameterization();
  lp->setParameter();
  lp->is_degenerate_ = true;
  lp->V_update_(0, 0) = 0.0;
  ceres::LocalParameterization *base = lp;
  double x[7] = {0, 0, 0, 0, 0, 0, 1}, d[6] = {0}, xp[7], J76[42];
  base->Plus(x, d, xp);
  base->ComputeJacobian(x, J76);

  const Eigen::Vector3d p(1, 2, 3);
  const Eigen::Vector4d c4(0, 0, 1, -1);
  Eigen::VectorXd c6(6);
  const Eigen::Matrix3d cov = Eigen::Matrix3d::Identity();
  ceres::CostFunction *fs[] = {new LidarMapPlaneNormFactor(p, c4, cov), new LidarMapEdgeFactor(p, c6, cov), new LidarScanPlaneNormFactor(p, c4, 1.0),
                               new LidarScanEdgeFactor(p, c6, 1.0), new LidarScanEdgeFactorVector(p, c6, 1.0), new LidarOnlineCalibPlaneNormFactor(p, c4, 1.0),
                               new LidarOnlineCalibEdgeFactor(p, c6, 1.0), new LidarPureOdomPlaneNormFactor(p, c4, 1.0), new LidarPureOdomEdgeFactor(p, c6, 1.0)};
  double r[3], j0[21], j1[7], j2[7];
  double *jac[3] = {j0, j1, j2};
  const double *params[3] = {x, x, x};
  int n = 0;
  for (ceres::CostFunction *f : fs) n += f->Evaluate(params, r, jac) ? 1 : 0;

  LidarTracker tracker;
  Pose out = tracker.trackCloud(feat, feat, pose_local);
  tracker.f_extract_.extractCloud(cloud, scan_info, feat);

  ActiveFeatureSelection afs;
  std::vector<size_t> sel;
  Eigen::Matrix<double, 6, 6> H;
  afs.goodFeatureMatching(kd_cov, cov_map, cov_scan, pose_local, features, sel, 's', "gd_float", 0.8, H);
  return n + (int)sel.size() + (int)out.t_(0);
}
