// TEST STUB — mloam_pcl/point_with_time.hpp (pcl::PointXYZIWithTime, common::PointITimeCloud), reduced to members; include guard as the real one.
#ifndef POINTWITHTIME_HPP
#define POINTWITHTIME_HPP
#include <pcl/point_cloud.h>

namespace pcl {
struct PointXYZIWithTime {
  float x = 0, y = 0, z = 0, pad0 = 1, intensity = 0, timestamp = 0, pad1[2] = {0, 0};
};
}  // namespace pcl
namespace common {
typedef pcl::PointXYZIWithTime PointIWithTime;
typedef pcl::PointCloud<PointIWithTime> PointITimeCloud;
}  // namespace common
#endif
