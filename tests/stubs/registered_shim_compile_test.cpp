// Compile check of the pubPointCloud wrappers of m-loam_b200/host/mloam_shim.hpp (plain g++, no third-party headers).  Compiled, never run:
// the frame calls need an H100.
#include "mloam_shim.hpp"

int shim_registered_use(mloam_ctx_t *ctx) {
  mloam::setRegistered(ctx, true);
  common::PointICloud laser_cloud_full_res, laser_cloud_surf_last, laser_cloud_corner_last;
  mloam::frameRegistered(ctx, laser_cloud_full_res, laser_cloud_surf_last, laser_cloud_corner_last);
  mloam::frameRegistered(ctx, MLOAM_REGISTERED_CORNER, laser_cloud_corner_last);
  return (int)(laser_cloud_full_res.size() + laser_cloud_surf_last.size() + laser_cloud_corner_last.size());
}
