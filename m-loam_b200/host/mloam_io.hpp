// mloam_io.hpp — wire formats either side of the hot path (SURVEY.md 8f item 4), host-only, no ROS / PCL needed:
//
//   sensor_msgs/PointCloud2 <-> mloam_point_t[]   the buffers the ROS nodes exchange (rosNodeRVHercules.cpp, lidar_mapper_keyframe.cpp
//                                                :1258-1277) packed into / out of the 16-byte float4 layout of the C ABI
//   mloam_msgs/Extrinsics, mloam_msgs/Keyframes   (mloam_msgs/msg/*.msg): header + status + odometry / pose-with-covariance arrays as PODs
//   TUM trajectory dump                          save_statistics.hpp:104-119: "stamp x y z qx qy qz qw", stamp with 15 significant
//                                                digits, the rest with 8 (std::ostream::precision semantics, not fixed notation)
//
// PointCloud2 layout rules implemented (sensor_msgs/PointCloud2 definition): fields are located by NAME ("x", "y", "z",
// "intensity"), each with its byte offset and datatype (FLOAT32 = 7; FLOAT64 = 8 is converted); a field lies inside the point (offset +
// size <= point_step); points are `point_step` bytes apart, rows `row_step` apart; is_bigendian data is byte-swapped; a missing
// "intensity" field gives 0 — the reference exits in that case (feature_extract.hpp:138-142), which callers can reproduce by checking
// PointCloud2View::has_intensity.  The fourth lane may name another field: "timestamp" for calTimestamp's PointITimeCloud overload.
// The device unpack of mloam_frame_msg* follows the same rules (resolvePointCloud2Layout).
#pragma once
#include <cstdint>
#include <cstring>
#include <ostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"

namespace mloam {
namespace io {

enum PointFieldType { INT8 = 1, UINT8 = 2, INT16 = 3, UINT16 = 4, INT32 = 5, UINT32 = 6, FLOAT32 = 7, FLOAT64 = 8 };

struct PointField {  // sensor_msgs/PointField
  std::string name;
  uint32_t offset = 0;
  uint8_t datatype = FLOAT32;
  uint32_t count = 1;
};

struct PointCloud2View {  // the members of sensor_msgs/PointCloud2 the packing needs (data is not owned)
  uint32_t height = 1, width = 0;
  std::vector<PointField> fields;
  bool is_bigendian = false;
  uint32_t point_step = 0, row_step = 0;
  const uint8_t *data = nullptr;
  size_t data_size = 0;
  bool has_intensity = false;  // set by unpack
  bool is_dense = false;       // no point is invalid (sensor_msgs/PointCloud2::is_dense); set by cloudMsgView
};

namespace detail {
inline float load_scalar(const uint8_t *p, uint8_t datatype, bool swap) {
  uint8_t b[8];
  const int n = datatype == FLOAT64 ? 8 : 4;
  for (int i = 0; i < n; i++) b[i] = swap ? p[n - 1 - i] : p[i];
  if (datatype == FLOAT64) {
    double d;
    std::memcpy(&d, b, 8);
    return (float)d;
  }
  float f;
  std::memcpy(&f, b, 4);
  return f;
}
inline bool host_is_bigendian() {
  const uint16_t one = 1;
  return *reinterpret_cast<const uint8_t *>(&one) == 0;
}
inline const PointField *find_field(const PointCloud2View &msg, const char *name) {
  if (!name) return nullptr;
  for (const PointField &f : msg.fields)
    if (f.name == name) return &f;
  return nullptr;
}
// FLOAT32 or FLOAT64, inside the point
inline bool field_ok(const PointField &f, uint32_t point_step) {
  if (f.datatype != FLOAT32 && f.datatype != FLOAT64) return false;
  return (uint64_t)f.offset + (f.datatype == FLOAT64 ? 8u : 4u) <= point_step;
}
}  // namespace detail

// PointCloud2 -> float4 points (x, y, z, lane 3); lane 3 is the field named lane3 ("intensity" by default, nullptr: none), 0 when the
// message has no such field.  Returns false when x / y / z are missing, a field is not FLOAT32 / FLOAT64 or does not lie inside the point
// (offset + size > point_step), or the buffer is shorter than height * row_step.
inline bool unpackPointCloud2(PointCloud2View &msg, std::vector<mloam_point_t> &out, const char *lane3 = "intensity") {
  const PointField *fx = detail::find_field(msg, "x"), *fy = detail::find_field(msg, "y"), *fz = detail::find_field(msg, "z");
  const PointField *fi = detail::find_field(msg, lane3);
  msg.has_intensity = detail::find_field(msg, "intensity") != nullptr;
  out.clear();
  if (!fx || !fy || !fz) return false;
  for (const PointField *f : {fx, fy, fz, fi})
    if (f && !detail::field_ok(*f, msg.point_step)) return false;
  const uint32_t row_step = msg.row_step ? msg.row_step : msg.width * msg.point_step;
  if (!msg.data || msg.data_size < (size_t)msg.height * row_step) return false;
  const bool swap = msg.is_bigendian != detail::host_is_bigendian();
  out.resize((size_t)msg.height * msg.width);
  size_t k = 0;
  for (uint32_t r = 0; r < msg.height; r++)
    for (uint32_t c = 0; c < msg.width; c++, k++) {
      const uint8_t *p = msg.data + (size_t)r * row_step + (size_t)c * msg.point_step;
      out[k].x = detail::load_scalar(p + fx->offset, fx->datatype, swap);
      out[k].y = detail::load_scalar(p + fy->offset, fy->datatype, swap);
      out[k].z = detail::load_scalar(p + fz->offset, fz->datatype, swap);
      out[k].intensity = fi ? detail::load_scalar(p + fi->offset, fi->datatype, swap) : 0.0f;
    }
  return true;
}

// The layout of msg's points for mloam_set_front_end_layout, found by field name once per driver: x, y, z and, with lane3 (e.g.
// "timestamp" for time_field 1), that field as lane 3; lane3 nullptr: no lane 3.  Returns false when x / y / z or the lane-3 field asked
// for are missing, a field is not FLOAT32 / FLOAT64, or a field does not lie inside the point (offset + size > point_step).
inline bool resolvePointCloud2Layout(const PointCloud2View &msg, const char *lane3, mloam_pc2_layout_t &layout) {
  const PointField *f[4] = {detail::find_field(msg, "x"), detail::find_field(msg, "y"), detail::find_field(msg, "z"),
                            detail::find_field(msg, lane3)};
  std::memset(&layout, 0, sizeof(layout));
  if (msg.point_step > 1024) return false;  // mloam_set_front_end_layout's bound
  for (int k = 0; k < 4; k++) {
    if (!f[k]) {
      if (k < 3 || lane3) return false;
      continue;
    }
    if (!detail::field_ok(*f[k], msg.point_step)) return false;
    layout.offset[k] = (int)f[k]->offset, layout.datatype[k] = f[k]->datatype;
  }
  layout.point_step = (int)msg.point_step, layout.is_bigendian = msg.is_bigendian ? 1 : 0;
  return true;
}

// One LiDAR's message for mloam_frame_msg* (the bytes stay the caller's)
inline mloam_pc2_msg_t pointCloud2Msg(const PointCloud2View &msg) {
  mloam_pc2_msg_t m;
  m.data = msg.data, m.size = msg.data_size, m.width = (int)msg.width, m.height = (int)msg.height;
  m.row_step = msg.row_step ? msg.row_step : (size_t)msg.width * msg.point_step;
  return m;
}

namespace detail {
// the fields pcl::toROSMsg lists for pcl::PointXYZI (n = 4) and mloam_pcl::PointXYZIWithCov (n = 11, point_with_cov.hpp:113-125)
inline std::vector<PointField> cloud_fields(int n) {
  static const char *const names[11] = {"x", "y", "z", "intensity", "cov_xx", "cov_xy", "cov_xz", "cov_yy", "cov_yz", "cov_zz", "cov_trace"};
  static const uint32_t offs[11] = {0, 4, 8, 16, 20, 24, 28, 32, 36, 40, 44};
  std::vector<PointField> fields(n);
  for (int i = 0; i < n; i++) fields[i].name = names[i], fields[i].offset = offs[i], fields[i].datatype = FLOAT32, fields[i].count = 1;
  return fields;
}
}  // namespace detail

// float4 points -> the PointCloud2 layout pcl::toROSMsg gives a pcl::PointXYZI cloud: point_step 32, x/y/z at 0/4/8, intensity at 16,
// unorganised (height 1), little endian.  `storage` receives the bytes the returned view points at.
inline PointCloud2View packPointCloud2(const mloam_point_t *pts, size_t n, std::vector<uint8_t> &storage) {
  PointCloud2View msg;
  msg.height = 1, msg.width = (uint32_t)n, msg.point_step = 32, msg.row_step = (uint32_t)(32 * n), msg.is_bigendian = false;
  msg.fields = detail::cloud_fields(4);
  storage.assign(32 * n, 0);
  for (size_t i = 0; i < n; i++) {
    std::memcpy(&storage[32 * i], &pts[i].x, 12);
    std::memcpy(&storage[32 * i + 16], &pts[i].intensity, 4);
  }
  msg.data = storage.data(), msg.data_size = storage.size(), msg.has_intensity = true;
  return msg;
}

// float4 points with cov_vec (6 floats per point: xx xy xz yy yz zz) and cov_trace -> the PointCloud2 layout pcl::toROSMsg gives a
// mloam_pcl::PointXYZIWithCov cloud: point_step 48, x/y/z at 0/4/8, intensity at 16, cov_xx .. cov_zz at 20 .. 40, cov_trace at 44,
// unorganised, little endian; bytes 12-15 are zero.  `storage` receives the bytes the returned view points at.
inline PointCloud2View packPointCloud2Cov(const mloam_point_t *pts, const float *cov6, const float *trace, size_t n,
                                          std::vector<uint8_t> &storage) {
  PointCloud2View msg;
  msg.height = 1, msg.width = (uint32_t)n, msg.point_step = 48, msg.row_step = (uint32_t)(48 * n), msg.is_bigendian = false;
  msg.fields = detail::cloud_fields(11);
  storage.assign(48 * n, 0);
  for (size_t i = 0; i < n; i++) {
    std::memcpy(&storage[48 * i], &pts[i].x, 12);
    std::memcpy(&storage[48 * i + 16], &pts[i].intensity, 4);
    std::memcpy(&storage[48 * i + 20], cov6 + 6 * i, 24);
    std::memcpy(&storage[48 * i + 44], trace + i, 4);
  }
  msg.data = storage.data(), msg.data_size = storage.size(), msg.has_intensity = true;
  return msg;
}

// point_step of a mloam_cloud_msgs* source: 32 (PointXYZI) or 48 (PointXYZIWithCov)
inline uint32_t cloudMsgStep(int source) { return source >= MLOAM_MSG_SURROUND ? 48u : 32u; }

// The PointCloud2 a message of mloam_cloud_msgs* is: `width` points of `source` (MLOAM_MSG_*) at data, its fields, steps and is_dense —
// false for MLOAM_MSG_FULL_RES, which holds the sweep's non-finite points, true for the others.  The bytes stay the caller's.
inline PointCloud2View cloudMsgView(int source, size_t width, const uint8_t *data) {
  PointCloud2View msg;
  msg.height = 1, msg.width = (uint32_t)width, msg.point_step = cloudMsgStep(source), msg.row_step = (uint32_t)(msg.point_step * width);
  msg.is_bigendian = false, msg.is_dense = source != MLOAM_MSG_FULL_RES;
  msg.fields = detail::cloud_fields(msg.point_step == 48 ? 11 : 4);
  msg.data = data, msg.data_size = (size_t)msg.point_step * width, msg.has_intensity = true;
  return msg;
}

// mloam_cloud_msgs of `sources` into data[k], each resized to its message (width[k] x cloudMsgStep bytes).  The buffers' capacities are
// offered first, so a caller that keeps its buffers from frame to frame pays one launch per call; a message that outgrew its buffer
// costs a second call.  Returns the library's code.
inline int cloudMsgs(mloam_ctx_t *ctx, const std::vector<int> &sources, std::vector<std::vector<uint8_t> *> &data, std::vector<int> &width) {
  const size_t n = sources.size();
  std::vector<void *> dst(n);
  std::vector<size_t> cap(n);
  width.assign(n, 0);
  int rc = MLOAM_OK;
  for (int pass = 0; pass < 2; pass++) {
    for (size_t k = 0; k < n; k++) {
      std::vector<uint8_t> &d = *data[k];
      d.resize(pass == 0 ? d.capacity() : (size_t)width[k] * cloudMsgStep(sources[k]));
      dst[k] = d.empty() ? nullptr : d.data(), cap[k] = d.size();
    }
    rc = mloam_cloud_msgs(ctx, (int)n, sources.data(), dst.data(), cap.data(), width.data());
    bool fit = true;
    for (size_t k = 0; k < n; k++) fit = fit && (size_t)width[k] * cloudMsgStep(sources[k]) <= cap[k];
    if (!fit && pass == 0) continue;  // too small (MLOAM_E_INVALID), or an empty buffer taken as a size query
    break;
  }
  for (size_t k = 0; k < n && rc == MLOAM_OK; k++) data[k]->resize((size_t)width[k] * cloudMsgStep(sources[k]));
  return rc;
}

// ---- mloam_msgs (header reduced to stamp + frame_id; nav_msgs/Odometry and PoseWithCovarianceStamped to what the nodes fill)
struct Header {
  double stamp = 0.0;
  std::string frame_id;
};
struct PoseWithCovariance {
  double position[3] = {0, 0, 0};
  double orientation[4] = {0, 0, 0, 1};  // x y z w
  double covariance[36] = {0};           // row-major 6x6 (geometry_msgs/PoseWithCovariance)
};
struct Odometry {  // nav_msgs/Odometry: header, child_frame_id, pose (twist unused by M-LOAM)
  Header header;
  std::string child_frame_id;
  PoseWithCovariance pose;
};
struct Extrinsics {  // mloam_msgs/Extrinsics.msg
  Header header;
  uint8_t status = 0;
  std::vector<Odometry> odoms;
};
struct PoseWithCovarianceStamped {
  Header header;
  PoseWithCovariance pose;
};
struct Keyframes {  // mloam_msgs/Keyframes.msg
  Header header;
  uint8_t status = 0;
  std::vector<PoseWithCovarianceStamped> poses;
};
// parameter block [tx ty tz qx qy qz qw] (pose_local_parameterization.h:20) <-> message pose
inline void poseFromParam(const double *x7, PoseWithCovariance &p) {
  for (int k = 0; k < 3; k++) p.position[k] = x7[k];
  for (int k = 0; k < 4; k++) p.orientation[k] = x7[3 + k];
}
inline void poseToParam(const PoseWithCovariance &p, double *x7) {
  for (int k = 0; k < 3; k++) x7[k] = p.position[k];
  for (int k = 0; k < 4; k++) x7[3 + k] = p.orientation[k];
}

// ---- TUM trajectory line / file (save_statistics.hpp:104-119)
inline void writeTumLine(std::ostream &os, double stamp, const double *x7) {
  os.precision(15);
  os << stamp << " ";
  os.precision(8);
  os << x7[0] << " " << x7[1] << " " << x7[2] << " " << x7[3] << " " << x7[4] << " " << x7[5] << " " << x7[6] << std::endl;
}
inline std::string tumTrajectory(const std::vector<double> &stamps, const std::vector<double> &poses7) {
  std::ostringstream os;
  for (size_t i = 0; i < stamps.size(); i++) writeTumLine(os, stamps[i], &poses7[7 * i]);
  return os.str();
}

}  // namespace io
}  // namespace mloam
