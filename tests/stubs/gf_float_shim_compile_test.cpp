// Compile check of ActiveFeatureSelection::evalFullHessian in m-loam_b200/host/mloam_shim.hpp (plain g++, no third-party headers):
// surf then corner into one mat_H, as lidar_mapper_keyframe.cpp:461-467.  Compiled, never run: the calls need an H100.
#include "mloam_shim.hpp"

int shim_eval_full_hessian() {
  common::PointICloud surf, corner;
  Pose pose_wmap_curr;
  ActiveFeatureSelection afs;
  int total_feat_num = 0;
  double mat_H[36] = {0};
  for (int i = 0; i < 6; i++) mat_H[i * 7] = 1e-6;
  afs.evalFullHessian(MLOAM_MAP_SURF, surf, pose_wmap_curr, 's', mat_H, total_feat_num);
  afs.evalFullHessian(MLOAM_MAP_CORNER, corner, pose_wmap_curr, 'c', mat_H, total_feat_num);
  return total_feat_num;
}
