// uct.h — the per-point association with uncertainty (cloudUCTAssociateToMap, lidar_mapper_keyframe.cpp:1116-1158) shared by the
// submap assembly (submap.cu) and the keyframe store (keyframe.cu).
#pragma once
#include <vector>

#include "ctx.h"

namespace mloam {

// UctLaser / UctFrame: ctx.h
// work of one association run over n points: k_uct_associate's staged points, cov_vec, trace and keep flags, the scan's slots + tmp,
// the kept count
struct UctBufs {
  float4 *staged;
  float *cov6, *trace;
  int *keep, *slot, *tmp, *count;
};
void uct_bufs_layout(Carve &cv, int n, UctBufs *B);
int uct_bufs(Ctx *c, int n, UctBufs *B);  // in Ctx::assoc_work()
// One keyframe cloud (device) -> associated + gated points appended at out[*d_total ...); *d_total advances on the device.
int uct_associate_append(Ctx *c, const float4 *d_pts, int n, const UctFrame &f, const UctLaser *d_lasers, const UctBufs &B, float4 *d_out,
                         float *d_cov6_out, float *d_trace_out, int *d_total);
// A run of one keyframe cloud in a batched association: points [begin, begin + n) of the concatenated input are pts[0, n), associated
// with keyframe kf's pose and UctLaser block
struct UctSeg {
  const float4 *pts;
  int begin, n, kf;
};
// n_seg non-empty segments in output order (n points in all) -> k_uct_associate_seg -> one exclusive scan of the keep flags -> one
// stable compaction into out / cov6_out / trace_out; the kept count lands in *B.count.  Five launches whatever the number of segments.
// f: cov_meas, trace_threshold, with_ua and n_lasers of every segment (pose_global unused); d_kf_pose7: 7 doubles per keyframe;
// d_lasers: f.n_lasers UctLaser per keyframe.
int uct_associate_segments(Ctx *c, const UctSeg *d_seg, int n_seg, int n, const UctFrame &f, const double *d_kf_pose7, const UctLaser *d_lasers,
                           const UctBufs &B, float4 *d_out, float *d_cov6_out, float *d_trace_out);
void fill_lasers(int n_lasers, const double *ext7, const double *pose_compound7, const double *cov_compound36, std::vector<UctLaser> &L);

}  // namespace mloam
