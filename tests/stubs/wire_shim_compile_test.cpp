// Compile check of the PointCloud2 message wrappers of m-loam_b200/host/mloam_shim.hpp (plain g++, no third-party headers).  Compiled,
// never run: the frame calls need an H100.
#include "mloam_shim.hpp"

int shim_wire_use(mloam_ctx_t *ctx, const std::vector<mloam::io::PointCloud2View> &msgs, const common::PointICloud &surf_map,
                  const common::PointICloud &corner_map) {
  mloam::setFrontEndLayout(ctx, msgs, true);
  Pose pose;
  mloam_solve_stats_t st;
  return mloam::frameMsg(ctx, msgs, surf_map, corner_map, pose, &st) ? st.n_surf : -1;
}
