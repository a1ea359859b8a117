// Relative time of a point inside its sweep: the arithmetic of FeatureExtract::calTimestamp (feature_extract.cpp:54-114), expression by
// expression.  atan2 on floats is the float overload there (parameters.h:43 `using namespace std`) — fdlibm atan2f here (fd_atan.cuh);
// SCAN_PERIOD is a float (parameters.h:78) and the M_PI expressions are doubles.  Explicitly rounded operations on the device, plain IEEE
// operations in a host build with -ffp-contract=off (tests/test_front_end_cpu.py compiles this header for the host and compares it with a
// libm restatement of the reference loop).
//
// The loop carries one flag, half_passed, but whether point i raises it depends on that point alone (its first-half angle): with i* the
// first point that raises it, points <= i* take the first-half branch and points > i* the second-half one.  So the times are computed in
// parallel from (first point, last point, i*), every one a min / max over indices.
#pragma once
#include "project.cuh"

// pcl::removeNaNFromPointCloud (the driver nodes, rosNodeRVKITTI.cpp:154-161, rosNodeRVOxford.cpp:170-177): non-finite x, y or z drops the point
FD_HD bool ts_finite(float4 p) {
#if defined(__CUDA_ARCH__)
  return isfinite(p.x) && isfinite(p.y) && isfinite(p.z);
#else
  return std::isfinite(p.x) && std::isfinite(p.y) && std::isfinite(p.z);
#endif
}

// findStartEndAngle (:54-70) on the first and last point of the (NaN-free) sweep
FD_HD void ts_start_end(float4 first, float4 last, float *start_ori, float *end_ori) {
  const float s = -fd::atan2f(first.y, first.x);
  float e = (float)FD_DADD((double)-fd::atan2f(last.y, last.x), 2 * M_PI);
  if ((double)FD_SUB(e, s) > 3 * M_PI) e = (float)FD_DSUB((double)e, 2 * M_PI);
  else if ((double)FD_SUB(e, s) < M_PI) e = (float)FD_DADD((double)e, 2 * M_PI);
  *start_ori = s, *end_ori = e;
}

// :82-94, half_passed == false.  *flips: this point sets half_passed (for the points after it)
FD_HD float ts_ori_first_half(float4 p, float start_ori, bool *flips) {
  float ori = -fd::atan2f(p.y, p.x);
  if ((double)ori < FD_DSUB((double)start_ori, M_PI / 2)) ori = (float)FD_DADD((double)ori, 2 * M_PI);
  else if ((double)ori > FD_DADD((double)start_ori, M_PI * 3 / 2)) ori = (float)FD_DSUB((double)ori, 2 * M_PI);
  *flips = (double)FD_SUB(ori, start_ori) > M_PI;
  return ori;
}

// :95-106, half_passed == true
FD_HD float ts_ori_second_half(float4 p, float end_ori) {
  float ori = -fd::atan2f(p.y, p.x);
  ori = (float)FD_DADD((double)ori, 2 * M_PI);
  if ((double)ori < FD_DSUB((double)end_ori, M_PI * 3 / 2)) ori = (float)FD_DADD((double)ori, 2 * M_PI);
  else if ((double)ori > FD_DADD((double)end_ori, M_PI / 2)) ori = (float)FD_DSUB((double)ori, 2 * M_PI);
  return ori;
}

// :107-108
FD_HD float ts_rel_time(float ori, float start_ori, float end_ori, float scan_period) {
  return FD_MUL(FD_DIV(FD_SUB(ori, start_ori), FD_SUB(end_ori, start_ori)), scan_period);
}

// the PointITimeCloud overload (:38-52): intensity = timestamp [us] * 1e-6, the timestamp carried in the point's w lane
FD_HD float ts_from_stamp(float timestamp_us) { return (float)FD_DMUL((double)timestamp_us, 1e-6); }

// Time of point i of a sweep given its start / end angles (ts_start_end) and the flip index i* (time_field == 0), or from its timestamp
FD_HD float ts_point_time_at(float4 p, int i, float start_ori, float end_ori, int flip_index, int time_field, float scan_period) {
  if (time_field) return ts_from_stamp(p.w);
  bool flips;
  const float ori = i <= flip_index ? ts_ori_first_half(p, start_ori, &flips) : ts_ori_second_half(p, end_ori);
  return ts_rel_time(ori, start_ori, end_ori, scan_period);
}
// ... given the first / last finite points instead of the angles
FD_HD float ts_point_time(float4 p, int i, float4 first, float4 last, int flip_index, int time_field, float scan_period) {
  float start_ori = 0.f, end_ori = 0.f;
  if (!time_field) ts_start_end(first, last, &start_ori, &end_ori);
  return ts_point_time_at(p, i, start_ori, end_ori, flip_index, time_field, scan_period);
}
