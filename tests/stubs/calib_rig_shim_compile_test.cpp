// Compile check of the rig calibration wrapper of m-loam_b200/host/mloam_shim.hpp (plain g++, no third-party headers).  Compiled, never
// run: the solve needs an H100.
#include "mloam_shim.hpp"

int shim_calib_rig_use(mloam_ctx_t *ctx) {
  std::vector<common::PointICloud> surf(3), corner(3);
  Pose pose_pivot, pose_i;
  std::vector<Pose> pose_ext(3), prior(3);
  std::vector<int> rows;
  const mloam_solve_stats_t st = mloam::calibRig(ctx, 0, surf, corner, pose_pivot, pose_i, pose_ext, &prior, 1.0, 1.0, 2, 4, true, &rows);
  return st.termination + (int)rows.size();
}
