// Compile check of the rig calibration wrapper and PriorFactor of m-loam_b200/host/mloam_adapter.hpp against the stub headers, with the
// problem of estimator.cpp:633-642, 670-787 on the RV rig (4 LiDARs, IDX_REF 0, PRIOR_FACTOR 1).  Compiled, never run: the solve needs an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_calib_rig_use(mloam_ctx_t *ctx) {
  std::vector<PointICloud> surf(4), corner(4);
  Pose pose_pivot, pose_i;
  std::vector<Pose> pose_ext(4);
  std::vector<int> rows;
  const mloam_solve_stats_t st = mloam::calibRig(ctx, 0, surf, corner, pose_pivot, pose_i, pose_ext, &pose_ext, 10.0, 10.0, 2, 4, false, &rows);
  // the reference's own problem assembly keeps compiling: PriorFactor(tbl_[n], qbl_[n], PRIOR_FACTOR_POS, PRIOR_FACTOR_ROT)
  PriorFactor f(pose_ext[1].t_, pose_ext[1].q_, 10.0, 10.0);
  double x[7] = {0, 0, 0, 0, 0, 0, 1}, r[6], J[42];
  const double *param[1] = {x};
  double *jac[1] = {J};
  const ceres::CostFunction &cf = f;
  return (int)cf.Evaluate(param, r, jac) + st.termination + (int)rows.size();
}
