// Compile check of the DISTORTION helpers of m-loam_b200/host/mloam_adapter.hpp against the stub headers, with the calls of
// Estimator::process (estimator.cpp:575-580).  Compiled, never run: the frame calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

int adapter_undistort_use(mloam_ctx_t *ctx, const Pose &pose_rlt_ref, const std::vector<Eigen::Quaterniond> &qbl_,
                          const std::vector<Eigen::Vector3d> &tbl_, size_t IDX_REF, int ESTIMATE_EXTRINSIC, float SCAN_PERIOD) {
  mloam::setDistortion(ctx, true, SCAN_PERIOD);
  std::vector<Pose> pose_undist = mloam::undistortPoses(pose_rlt_ref, qbl_, tbl_);
  mloam::undistortMeasurements(ctx, pose_undist, IDX_REF, ESTIMATE_EXTRINSIC);
  return (int)pose_undist.size();
}
