// Compile check of the pubPointCloud wrappers of m-loam_b200/host/mloam_adapter.hpp against the stub headers, with the clouds of
// lidar_mapper_keyframe.cpp:690-714.  Compiled, never run: the frame calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_registered_use(mloam_ctx_t *ctx) {
  mloam::setRegistered(ctx, true);
  PointICloud laser_cloud_full_res, laser_cloud_surf_last, laser_cloud_corner_last;
  mloam::frameRegistered(ctx, laser_cloud_full_res, laser_cloud_surf_last, laser_cloud_corner_last);
  mloam::frameRegistered(ctx, MLOAM_REGISTERED_SURF, laser_cloud_surf_last);
  return (int)(laser_cloud_full_res.size() + laser_cloud_surf_last.size() + laser_cloud_corner_last.size());
}
