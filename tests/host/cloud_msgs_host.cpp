// Host build of m-loam_b200/host/mloam_io.hpp for tests/cloud_msgs_lib.py: packPointCloud2 / packPointCloud2Cov (the host statement of
// the layouts mloam_cloud_msgs* packs on the device) and the header cloudMsgView gives each source's message.
#include "mloam_io.hpp"

using namespace mloam::io;

// the bytes of packPointCloud2 (32 n) / packPointCloud2Cov (48 n) into out
extern "C" void cm_pack(const float *pts, size_t n, uint8_t *out) {
  std::vector<uint8_t> s;
  const PointCloud2View v = packPointCloud2(reinterpret_cast<const mloam_point_t *>(pts), n, s);
  if (v.data_size) std::memcpy(out, v.data, v.data_size);
}
extern "C" void cm_pack_cov(const float *pts, const float *cov6, const float *trace, size_t n, uint8_t *out) {
  std::vector<uint8_t> s;
  const PointCloud2View v = packPointCloud2Cov(reinterpret_cast<const mloam_point_t *>(pts), cov6, trace, n, s);
  if (v.data_size) std::memcpy(out, v.data, v.data_size);
}

// cloudMsgView(source, width): hdr = {height, width, point_step, row_step, is_bigendian, is_dense, n_fields}; per field its name (16
// bytes each), offset, datatype and count.  Returns the field count.
extern "C" int cm_view(int source, size_t width, int *hdr, char *names, int *offsets, int *datatypes, int *counts) {
  const PointCloud2View v = cloudMsgView(source, width, nullptr);
  const int nf = (int)v.fields.size();
  const int h[7] = {(int)v.height, (int)v.width, (int)v.point_step, (int)v.row_step, v.is_bigendian ? 1 : 0, v.is_dense ? 1 : 0, nf};
  std::memcpy(hdr, h, sizeof(h));
  for (int k = 0; k < nf; k++) {
    std::strncpy(names + 16 * k, v.fields[k].name.c_str(), 15);
    offsets[k] = (int)v.fields[k].offset, datatypes[k] = v.fields[k].datatype, counts[k] = (int)v.fields[k].count;
  }
  return nf;
}
