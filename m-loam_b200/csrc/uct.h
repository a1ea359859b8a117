// uct.h — the per-point association with uncertainty (cloudUCTAssociateToMap, lidar_mapper_keyframe.cpp:1116-1158) shared by the
// submap assembly (submap.cu) and the keyframe store (keyframe.cu).
#pragma once
#include <vector>

#include "ctx.h"

namespace mloam {

struct UctLaser {      // per LiDAR of the rig
  double ext_inv[7];   // pose_ext[n].inverse()
  double compound[7];  // pose_global * pose_ext[n]
  double cov[36];      // its covariance (compoundPoseWithCov)
};
struct UctFrame {
  double pose_global[7];
  double cov_meas[9];
  double trace_threshold;
  int with_ua, n_lasers;
  int scan_frame;  // 1: the scan of a with_ua frame (downsampleCurrentScan, lidar_mapper_keyframe.cpp:376-387): no pose_global transform
};

// device buffers of one association run inside scratch[2]
struct UctBufs {
  float4 *staged;
  float *cov6, *trace;
  int *keep, *slot, *tmp, *count;
};
int uct_bufs(Ctx *c, int n, UctBufs *B);
// One keyframe cloud (device) -> associated + gated points appended at out[*d_total ...); *d_total advances on the device.
int uct_associate_append(Ctx *c, const float4 *d_pts, int n, const UctFrame &f, const UctLaser *d_lasers, const UctBufs &B, float4 *d_out,
                         float *d_cov6_out, float *d_trace_out, int *d_total);
void fill_lasers(int n_lasers, const double *ext7, const double *pose_compound7, const double *cov_compound36, std::vector<UctLaser> &L);

}  // namespace mloam
