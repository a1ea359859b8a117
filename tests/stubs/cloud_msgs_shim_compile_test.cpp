// Compile check of the published-cloud message wrapper of m-loam_b200/host/mloam_shim.hpp (plain g++, no third-party headers).
// Compiled, never run: the calls need an H100.
#include "mloam_shim.hpp"

int shim_cloud_msgs_use(mloam_ctx_t *ctx) {
  std::vector<std::vector<uint8_t>> storage;
  const std::vector<mloam::io::PointCloud2View> msgs =
      mloam::cloudMsgs(ctx, {MLOAM_MSG_FULL_RES, MLOAM_MSG_SURF_LAST, MLOAM_MSG_CORNER_LAST, MLOAM_MSG_SURROUND}, storage);
  return (int)(msgs[0].width + msgs[3].point_step + (msgs[1].is_dense ? 1 : 0));
}
