// Compile check of ActiveFeatureSelection::evalFullHessian in m-loam_b200/host/mloam_adapter.hpp against the stub third-party headers in
// this directory, with the reference's call shape (lidar_mapper_keyframe.cpp:461-470).  Compiled, never run: the calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_eval_full_hessian() {
  mloam::KdTreeFLANN<PointIWithCov>::Ptr kdtree_surf_from_map(new mloam::KdTreeFLANN<PointIWithCov>());
  mloam::KdTreeFLANN<PointIWithCov>::Ptr kdtree_corner_from_map(new mloam::KdTreeFLANN<PointIWithCov>());
  PointICovCloud surf_map, corner_map, surf_cov, corner_cov;
  Pose pose_wmap_curr;
  ActiveFeatureSelection afs;
  int total_feat_num = 0;
  Eigen::Matrix<double, 6, 6> mat_H = Eigen::Matrix<double, 6, 6>::Identity();  // * 1e-6 in the reference; the stand-in has no product
  for (int i = 0; i < 6; i++) mat_H(i, i) = 1e-6;
  afs.evalFullHessian(kdtree_surf_from_map, surf_map, surf_cov, pose_wmap_curr, 's', mat_H, total_feat_num);
  afs.evalFullHessian(kdtree_corner_from_map, corner_map, corner_cov, pose_wmap_curr, 'c', mat_H, total_feat_num);
  return total_feat_num + (int)mat_H(0, 0);
}
