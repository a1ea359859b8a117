// Host build of m-loam_b200/host/mloam_io.hpp for tests/wire_lib.py: unpackPointCloud2 and resolvePointCloud2Layout over a message given
// as plain arrays (field names, offsets, datatypes), the host statement of the PointCloud2 rules the device unpack of mloam_frame_msg* follows.
#include "mloam_io.hpp"

using namespace mloam::io;

namespace {
PointCloud2View view(const uint8_t *data, size_t size, int width, int height, size_t row_step, int point_step, int is_bigendian, int n_fields,
                     const char *const *names, const int *offsets, const int *datatypes) {
  PointCloud2View m;
  m.data = data, m.data_size = size, m.width = (uint32_t)width, m.height = (uint32_t)height, m.row_step = (uint32_t)row_step;
  m.point_step = (uint32_t)point_step, m.is_bigendian = is_bigendian != 0;
  for (int k = 0; k < n_fields; k++) {
    PointField f;
    f.name = names[k], f.offset = (uint32_t)offsets[k], f.datatype = (uint8_t)datatypes[k];
    m.fields.push_back(f);
  }
  return m;
}
}  // namespace

// 1: out (width x height points) holds the unpacked cloud; 0: unpackPointCloud2 refused the message.  lane3 nullptr: the default ("intensity")
extern "C" int wire_unpack(const uint8_t *data, size_t size, int width, int height, size_t row_step, int point_step, int is_bigendian, int n_fields,
                           const char *const *names, const int *offsets, const int *datatypes, const char *lane3, float *out) {
  PointCloud2View m = view(data, size, width, height, row_step, point_step, is_bigendian, n_fields, names, offsets, datatypes);
  std::vector<mloam_point_t> pts;
  const bool ok = lane3 ? unpackPointCloud2(m, pts, lane3) : unpackPointCloud2(m, pts);
  if (ok) std::memcpy(out, pts.data(), sizeof(mloam_point_t) * pts.size());
  return ok ? 1 : 0;
}

// 1: *layout holds the resolved layout; 0: resolvePointCloud2Layout refused the fields.  lane3 nullptr: no lane 3
extern "C" int wire_layout(int point_step, int is_bigendian, int n_fields, const char *const *names, const int *offsets, const int *datatypes,
                           const char *lane3, mloam_pc2_layout_t *layout) {
  PointCloud2View m = view(nullptr, 0, 0, 1, 0, point_step, is_bigendian, n_fields, names, offsets, datatypes);
  return resolvePointCloud2Layout(m, lane3, *layout) ? 1 : 0;
}
