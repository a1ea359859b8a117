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
//
// PCD files (resolvePCDHeader, decodePCDASCII, pcdBinaryMsg): the header and body rules of pcl::io::loadPCDFile<pcl::PointXYZ>, below.
#pragma once
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <locale>
#include <ostream>
#include <sstream>
#include <string>
#include <vector>

#include "../../include/mloam_b200.h"
#include "../csrc/pcd_ascii.cuh"

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

// ---- PCD files: what the dataset nodes read per frame and LiDAR with pcl::io::loadPCDFile<pcl::PointXYZ>(cloud_<j>/data/<idx>.pcd)
// (rosNodeRVOxford.cpp:355-370, rosNodeRVHercules.cpp:354-368), written by pcl::io::savePCDFileASCII (test_parse_bag.cpp:47-72).
// Header: the v0.7 header PCL writes, `#` comment lines, then VERSION, FIELDS, SIZE, TYPE, COUNT (optional: 1 each), WIDTH, HEIGHT,
// VIEWPOINT, POINTS (optional: WIDTH x HEIGHT), DATA.  x, y and z must be fields of SIZE 4, TYPE F, COUNT 1 (what loadPCDFile<PointXYZ>
// maps by name); every other field, `_` padding included, only takes its COUNT tokens (ASCII) or SIZE x COUNT bytes (binary).  DATA ascii
// and binary are taken; binary_compressed and anything else are refused.
struct PCDLayout {
  int points = 0;                  // POINTS
  size_t body = 0;                 // byte offset of the body: the byte after the DATA line
  int tokens = 0;                  // ASCII: tokens per line (the fields' COUNTs summed)
  int index[3] = {0, 0, 0};        // ASCII: token index of x, y, z in a line
  bool binary = false;             // DATA binary
  int point_step = 0;              // binary: bytes per point (SIZE x COUNT summed)
  int offset[3] = {0, 0, 0};       // binary: byte offset of x, y, z in a point
};

namespace detail {
inline std::vector<std::string> pcd_split(const std::string &line) {
  std::vector<std::string> t;
  std::istringstream is(line);
  std::string w;
  while (is >> w) t.push_back(w);
  return t;
}
inline bool pcd_int(const std::string &s, long long &v) {
  if (s.empty()) return false;
  char *end = nullptr;
  v = std::strtoll(s.c_str(), &end, 10);
  return end && *end == '\0';
}
}  // namespace detail

// The header of the PCD file bytes[0, size) -> layout.  Returns false for a header this library does not take (see above), a missing
// or inconsistent FIELDS / SIZE / TYPE / COUNT, POINTS other than WIDTH x HEIGHT, or no DATA line.
inline bool resolvePCDHeader(const uint8_t *bytes, size_t size, PCDLayout &layout) {
  layout = PCDLayout{};
  std::vector<std::string> fields, sizes, types, counts;
  long long width = -1, height = -1, points = -1;
  size_t at = 0;
  while (at < size) {
    size_t end = at;
    while (end < size && bytes[end] != '\n') end++;
    const std::string line(reinterpret_cast<const char *>(bytes) + at, end - at);
    at = end < size ? end + 1 : end;
    const std::vector<std::string> t = detail::pcd_split(line);
    if (t.empty() || t[0][0] == '#') continue;
    const std::string &key = t[0];
    const std::vector<std::string> vals(t.begin() + 1, t.end());
    if (key == "VERSION" || key == "VIEWPOINT") continue;
    if (key == "FIELDS" || key == "COLUMNS") fields = vals;
    else if (key == "SIZE") sizes = vals;
    else if (key == "TYPE") types = vals;
    else if (key == "COUNT") counts = vals;
    else if (key == "WIDTH" || key == "HEIGHT" || key == "POINTS") {
      long long v;
      if (vals.size() != 1 || !detail::pcd_int(vals[0], v) || v < 0) return false;
      (key == "WIDTH" ? width : key == "HEIGHT" ? height : points) = v;
    } else if (key == "DATA") {
      if (vals.size() != 1 || (vals[0] != "ascii" && vals[0] != "binary")) return false;  // binary_compressed: refused
      layout.binary = vals[0] == "binary";
      layout.body = at;
      break;
    } else {
      return false;
    }
  }
  if (layout.body == 0 || fields.empty() || sizes.size() != fields.size() || types.size() != fields.size()) return false;
  if (counts.empty()) counts.assign(fields.size(), "1");
  if (counts.size() != fields.size() || width < 0 || height < 0) return false;
  if (points < 0) points = width * height;
  if (points != width * height || points > (1ll << 30)) return false;
  int found = 0;
  long long tok = 0, off = 0;
  for (size_t f = 0; f < fields.size(); f++) {
    long long sz, cnt;
    if (!detail::pcd_int(sizes[f], sz) || !detail::pcd_int(counts[f], cnt) || sz <= 0 || cnt <= 0 || types[f].size() != 1) return false;
    const int k = fields[f] == "x" ? 0 : fields[f] == "y" ? 1 : fields[f] == "z" ? 2 : -1;
    if (k >= 0) {
      if (sz != 4 || types[f] != "F" || cnt != 1 || (found & (1 << k))) return false;
      found |= 1 << k;
      layout.index[k] = (int)tok, layout.offset[k] = (int)off;
    }
    tok += cnt, off += sz * cnt;
    if (tok > (1 << 20) || off > (1 << 20)) return false;
  }
  if (found != 7) return false;
  layout.points = (int)points, layout.tokens = (int)tok, layout.point_step = (int)off;
  return true;
}

// A DATA binary body as the PointCloud2 message mloam_frame_msg* take: one row of POINTS points, point_step bytes each, x / y / z
// FLOAT32 at their offsets, no lane 3, little endian (PCL writes the host's byte order).  The bytes stay the caller's.  Returns false for
// an ASCII layout or a body shorter than POINTS x point_step.
inline bool pcdBinaryMsg(const uint8_t *bytes, size_t size, const PCDLayout &h, mloam_pc2_layout_t &layout, mloam_pc2_msg_t &msg) {
  std::memset(&layout, 0, sizeof(layout));
  std::memset(&msg, 0, sizeof(msg));
  if (!h.binary || h.body > size || (size - h.body) / (size_t)h.point_step < (size_t)h.points || h.point_step > 1024) return false;
  layout.point_step = h.point_step;
  for (int k = 0; k < 3; k++) layout.offset[k] = h.offset[k], layout.datatype[k] = FLOAT32;
  msg.data = bytes + h.body, msg.size = (size_t)h.points * h.point_step, msg.width = h.points, msg.height = 1;
  msg.row_step = (size_t)h.points * h.point_step;
  return true;
}

// One LiDAR's ASCII body for mloam_pcd_decode* / mloam_frame_pcd* (the bytes stay the caller's)
inline mloam_pcd_t pcdBody(const uint8_t *bytes, size_t size, const PCDLayout &h) {
  mloam_pcd_t p;
  std::memset(&p, 0, sizeof(p));
  p.data = bytes + h.body, p.size = size - h.body, p.points = h.points, p.tokens = h.tokens;
  for (int k = 0; k < 3; k++) p.index[k] = h.index[k];
  return p;
}

namespace detail {
// The bytes of the file at path, or false
inline bool read_file(const std::string &path, std::vector<uint8_t> &bytes) {
  std::FILE *f = std::fopen(path.c_str(), "rb");
  if (!f) return false;
  bytes.clear();
  uint8_t buf[1 << 16];
  size_t n;
  while ((n = std::fread(buf, 1, sizeof(buf), f)) > 0) bytes.insert(bytes.end(), buf, buf + n);
  const bool ok = std::ferror(f) == 0;
  std::fclose(f);
  return ok;
}
}  // namespace detail

// The ASCII body[0, size) -> POINTS float4 points (x, y, z, 0) in file order, as loadPCDFile<PointXYZ> reads them (PCL 1.8
// PCDReader::read, copyStringValue<float>), with std::istringstream and atof exactly as PCL calls them.  The rules:
//  - lines end at '\n'; a line that is empty or holds only spaces, tabs and '\r' is skipped (PCL skips only an empty line and throws on
//    the others);
//  - tokens are split on runs of space, tab and '\r', the line trimmed first; point i is the i-th line not skipped; lines after POINTS,
//    and tokens after the header's count on a line, are ignored;
//  - a token is "nan" (quiet NaN) or the float istringstream >> f reads, (float)atof(tok) when that read fails.
// Returns 0, or the PCD_E_* bits (csrc/pcd_ascii.cuh) of why the body is refused: a line with fewer tokens than the header's, fewer lines
// than POINTS, an x / y / z token outside pcd_ascii.cuh's grammar or with more than 19 significant digits.  The first refusal ends the
// decode.  Non-finite coordinates are passed on.
inline int decodePCDASCII(const uint8_t *body, size_t size, int points, int tokens, const int index[3], std::vector<mloam_point_t> &out) {
  out.assign((size_t)(points > 0 ? points : 0), mloam_point_t{0.f, 0.f, 0.f, 0.f});
  int idx = 0;
  size_t at = 0;
  std::vector<std::string> st;
  while (at < size && idx < points) {
    size_t end = at;
    while (end < size && body[end] != '\n') end++;
    const size_t a = at;
    at = end < size ? end + 1 : end;
    st.clear();
    for (size_t k = a; k < end;) {
      while (k < end && pcd::is_sep(body[k])) k++;
      const size_t t0 = k;
      while (k < end && !pcd::is_sep(body[k])) k++;
      if (k > t0) st.emplace_back(reinterpret_cast<const char *>(body) + t0, k - t0);
    }
    if (st.empty()) continue;
    if ((int)st.size() < tokens) return pcd::PCD_E_SHORT_LINE;
    float v[3];
    for (int c = 0; c < 3; c++) {
      const std::string &tok = st[(size_t)index[c]];
      uint32_t bits;
      const int ts = pcd::parse_float(reinterpret_cast<const unsigned char *>(tok.data()), (long long)tok.size(), &bits);
      if (ts != pcd::PCD_OK) return ts << 1;
      if (tok == "nan") {
        v[c] = std::numeric_limits<float>::quiet_NaN();
      } else {
        std::istringstream is(tok);
        is.imbue(std::locale::classic());
        if (!(is >> v[c])) v[c] = static_cast<float>(std::atof(tok.c_str()));
      }
    }
    out[(size_t)idx++] = mloam_point_t{v[0], v[1], v[2], 0.f};
  }
  return idx < points ? pcd::PCD_E_FEW_LINES : 0;
}

// The points of the PCD file at path (x, y, z, 0), for the adapter's and the shim's loadPCDFile: the header read here, an ASCII body
// decoded on the device by mloam_pcd_decode (the one helper of this header that calls the library), a binary one copied from its
// PointCloud2 layout.  false: the file cannot be read, or is refused.
inline bool loadPCDPoints(mloam_ctx_t *ctx, const std::string &path, std::vector<mloam_point_t> &pts) {
  std::vector<uint8_t> bytes;
  PCDLayout h;
  if (!detail::read_file(path, bytes) || !resolvePCDHeader(bytes.data(), bytes.size(), h)) return false;
  pts.assign((size_t)h.points, mloam_point_t{0.f, 0.f, 0.f, 0.f});
  if (h.binary) {
    mloam_pc2_layout_t lay;
    mloam_pc2_msg_t m;
    if (!pcdBinaryMsg(bytes.data(), bytes.size(), h, lay, m)) return false;
    for (size_t i = 0; i < pts.size(); i++) {
      const uint8_t *p = static_cast<const uint8_t *>(m.data) + i * (size_t)lay.point_step;
      std::memcpy(&pts[i].x, p + lay.offset[0], 4), std::memcpy(&pts[i].y, p + lay.offset[1], 4), std::memcpy(&pts[i].z, p + lay.offset[2], 4);
    }
    return true;
  }
  if (h.points == 0) return true;
  const mloam_pcd_t body = pcdBody(bytes.data(), bytes.size(), h);
  return mloam_pcd_decode(ctx, 1, &body, pts.data()) == MLOAM_OK;
}

// ---- PCD files written: pcl::PCDWriter::write(file, cloud) = writeASCII(file, cloud, 8) (PCL 1.8.0 pcd_io.hpp) of saveGlobalMap
// (lidar_mapper_keyframe.cpp:853-919) and pcl::io::savePCDFileASCII (test_parse_bag.cpp:47-72); the format is stated with
// mloam_cloud_pcd in include/mloam_b200.h.  The fields of a layout: pcdFields(MLOAM_PCD_*).
inline int pcdFields(int layout) { return layout == MLOAM_PCD_XYZ ? 3 : layout == MLOAM_PCD_XYZI ? 4 : 11; }

// PCL's writer restated with an ostringstream, precision 8, the classic locale and the pcl_isnan test: the file of n points (pts; cov6 /
// trace for MLOAM_PCD_XYZI_COV).  An empty cloud gives "" (PCL throws and writes nothing).
inline std::string writePCDASCII(int layout, const mloam_point_t *pts, const float *cov6, const float *trace, size_t n) {
  if (n == 0) return std::string();
  static const char *const names[11] = {"x", "y", "z", "intensity", "cov_xx", "cov_xy", "cov_xz", "cov_yy", "cov_yz", "cov_zz", "cov_trace"};
  const int nf = pcdFields(layout);
  std::ostringstream os;
  os.imbue(std::locale::classic());
  os << "# .PCD v0.7 - Point Cloud Data file format\nVERSION 0.7\nFIELDS";
  for (int f = 0; f < nf; f++) os << " " << names[f];
  os << "\nSIZE";
  for (int f = 0; f < nf; f++) os << " 4";
  os << "\nTYPE";
  for (int f = 0; f < nf; f++) os << " F";
  os << "\nCOUNT";
  for (int f = 0; f < nf; f++) os << " 1";
  os << "\nWIDTH " << n << "\nHEIGHT 1\nVIEWPOINT 0 0 0 1 0 0 0\nPOINTS " << n << "\nDATA ascii\n";
  os.precision(8);
  for (size_t i = 0; i < n; i++) {
    const float v[11] = {pts[i].x, pts[i].y, pts[i].z, pts[i].intensity, cov6 ? cov6[6 * i] : 0.f, cov6 ? cov6[6 * i + 1] : 0.f,
                         cov6 ? cov6[6 * i + 2] : 0.f, cov6 ? cov6[6 * i + 3] : 0.f, cov6 ? cov6[6 * i + 4] : 0.f,
                         cov6 ? cov6[6 * i + 5] : 0.f, trace ? trace[i] : 0.f};
    for (int f = 0; f < nf; f++) {
      if (f) os << " ";
      if (v[f] != v[f]) os << "nan";
      else os << v[f];
    }
    os << "\n";
  }
  return os.str();
}

// mloam_cloud_pcd of `sources` into data[k], each resized to its file.  The buffers' capacities are offered first, so a caller that keeps
// its buffers pays one launch per call; a file that outgrew its buffer costs a second call.  Returns the library's code.
inline int cloudPCD(mloam_ctx_t *ctx, const std::vector<int> &sources, std::vector<std::vector<uint8_t> *> &data) {
  const size_t n = sources.size();
  std::vector<void *> dst(n);
  std::vector<size_t> cap(n), bytes(n, 0);
  int rc = MLOAM_OK;
  for (int pass = 0; pass < 2; pass++) {
    for (size_t k = 0; k < n; k++) {
      std::vector<uint8_t> &d = *data[k];
      d.resize(pass == 0 ? d.capacity() : bytes[k]);
      dst[k] = d.empty() ? nullptr : d.data(), cap[k] = d.size();
    }
    rc = mloam_cloud_pcd(ctx, (int)n, sources.data(), dst.data(), cap.data(), bytes.data());
    bool fit = true;
    for (size_t k = 0; k < n; k++) fit = fit && bytes[k] <= cap[k];
    if (!fit && pass == 0) continue;  // too small (MLOAM_E_INVALID), or an empty buffer taken as a size query
    break;
  }
  for (size_t k = 0; k < n && rc == MLOAM_OK; k++) data[k]->resize(bytes[k]);
  return rc;
}

// The file bytes at path; false when it cannot be written
inline bool savePCD(const std::string &path, const std::vector<uint8_t> &bytes) {
  std::FILE *f = std::fopen(path.c_str(), "wb");
  if (!f) return false;
  const bool ok = std::fwrite(bytes.data(), 1, bytes.size(), f) == bytes.size();
  return std::fclose(f) == 0 && ok;
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
