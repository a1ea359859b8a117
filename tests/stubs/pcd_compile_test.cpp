// Compile check of the PCD loader of m-loam_b200/host/mloam_adapter.hpp (pcl::PointCloud<pcl::PointXYZ>), as the dataset nodes call
// loadPCDFile per frame and LiDAR (plain g++, stand-in PCL headers).  Compiled, never run: the decode needs an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>
#include "reference_types.h"
#include "common/types/type.h"
#include "../../m-loam_b200/host/mloam_adapter.hpp"

int pcd_use(mloam_ctx_t *ctx, const std::string &path) {
  pcl::PointCloud<pcl::PointXYZ> cloud;
  return mloam::loadPCDFile(ctx, path, cloud) == -1 ? -1 : (int)cloud.size();
}
