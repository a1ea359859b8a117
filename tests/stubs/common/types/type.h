// TEST STUB — the part of mloam_common's common/types/type.h the calTimestamp adapter needs: common::PointCloud of pcl::PointXYZ.
#pragma once
#include <pcl/point_cloud.h>

namespace pcl {
struct PointXYZ {
  float x = 0, y = 0, z = 0, pad0 = 1;
};
}  // namespace pcl
namespace common {
typedef pcl::PointXYZ Point;
typedef pcl::PointCloud<Point> PointCloud;
}  // namespace common
