// Host build of m-loam_b200/host/mloam_adapter.hpp's PriorFactor against the stub headers, for tests/test_calib_rig_cpu.py: its residual
// and 6 x 7 Jacobian at x7 with target x07.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

extern "C" void host_prior_factor(const double *x7, const double *x07, double pos_scale, double rot_scale, double *r6, double *J42) {
  const PriorFactor f(Eigen::Vector3d(x07[0], x07[1], x07[2]), Eigen::Quaterniond(x07[6], x07[3], x07[4], x07[5]), pos_scale, rot_scale);
  const double *param[1] = {x7};
  double *jac[1] = {J42};
  f.Evaluate(param, r6, jac);
}
