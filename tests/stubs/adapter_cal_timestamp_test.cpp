// Compile check of FeatureExtract::calTimestamp in m-loam_b200/host/mloam_adapter.hpp against the stub headers: both reference overloads
// (feature_extract.hpp:68-72) with the calls of Estimator::inputCloud (estimator.cpp:252) on a PointCloud and on a PointITimeCloud.
// Compiled and linked against libmloam_b200.so, never run: the calls need an H100.
#include <Eigen/Dense>
#include <ceres/ceres.h>
#include <pcl/point_cloud.h>
#include <pcl/point_types.h>

#include "common/types/type.h"
#include "mloam_pcl/point_with_time.hpp"
#include "reference_types.h"

#include "../../m-loam_b200/host/mloam_adapter.hpp"

double ROI_RANGE = 0.5;
float SCAN_PERIOD = 0.1f;

int adapter_cal_timestamp_use() {
  FeatureExtract f_extract;
  common::PointCloud xyz;
  common::PointITimeCloud timed;
  PointICloud out;
  f_extract.calTimestamp(xyz, out);
  f_extract.calTimestamp(timed, out);
  return (int)out.size();
}
