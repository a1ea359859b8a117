// Compile check of the PCD loader of m-loam_b200/host/mloam_shim.hpp (float4 points; plain g++, no third-party headers).  Compiled,
// never run: the decode needs an H100.
#include "mloam_shim.hpp"

int shim_pcd_use(mloam_ctx_t *ctx, const std::string &path) {
  std::vector<mloam_point_t> pts;
  return mloam::loadPCDFile(ctx, path, pts) == -1 ? -1 : (int)pts.size();
}
