// Compile check of the PCD writers of m-loam_b200/host/mloam_adapter.hpp against the stub headers, with the calls of saveGlobalMap
// (lidar_mapper_keyframe.cpp:853-919) and test_parse_bag.cpp:47-72.  Compiled, never run: the writes need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int pcd_write_use(mloam_ctx_t *ctx, const pcl::PointCloud<pcl::PointXYZ> &sweep, const pcl::PointCloud<pcl::PointXYZI> &pose_keyframes_3d,
                  const pcl::PointCloud<pcl::PointXYZIWithCov> &laser_cloud_surf_map_ds) {
  mloam::PCDWriter pcd_writer(ctx);
  int rc = pcd_writer.write("/tmp/mloam_mapping_keyframes.pcd", pose_keyframes_3d);
  rc |= pcd_writer.write("/tmp/mloam_mapping_surf_cloud.pcd", laser_cloud_surf_map_ds);
  rc |= mloam::savePCDFileASCII(ctx, "cloud_0/data/0.pcd", sweep);
  return rc | mloam::saveGlobalMap(ctx, "/tmp/", true, 0.4f);
}
