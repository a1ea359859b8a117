// Minimal stand-in for the ROS message header sensor_msgs/PointCloud2.h (with sensor_msgs/PointField): the members of the real messages,
// so that m-loam_b200/host/mloam_adapter.hpp's toROSMsg wrapper is compile-checked without ROS.
#pragma once
#include <cstdint>
#include <string>
#include <vector>

namespace std_msgs {
struct Header {
  uint32_t seq = 0;
  struct {
    uint32_t sec = 0, nsec = 0;
  } stamp;
  std::string frame_id;
};
}  // namespace std_msgs

namespace sensor_msgs {
struct PointField {
  enum { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = 0;
  uint32_t count = 0;
};
struct PointCloud2 {
  std_msgs::Header header;
  uint32_t height = 0, width = 0;
  std::vector<PointField> fields;
  uint8_t is_bigendian = 0;
  uint32_t point_step = 0, row_step = 0;
  std::vector<uint8_t> data;
  uint8_t is_dense = 0;
};
}  // namespace sensor_msgs
