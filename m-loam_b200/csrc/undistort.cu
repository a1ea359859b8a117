// undistort.cu — the DISTORTION step of the odometry (estimator.cpp:545-590 -> undistortMeasurements :376-408 -> TransformToEnd,
// utility.h:54-100) in the frame path:
//   mloam_undistort_poses   pose_undist[n] = ext_n^-1 * pose_rlt[IDX_REF] * ext_n (pose.cpp:99-102, 110-113), and which of them each
//                           LiDAR's features move with (ESTIMATE_EXTRINSIC == 2: its own; otherwise IDX_REF's, :403-405) — host only
//   mloam_set_distortion    on / off and SCAN_PERIOD
//   mloam_frame_undistort   the per-LiDAR poses of the sweep of the next mloam_frame* call
//   mloam_frame_set_next_undistort   the poses of the sweep announced for the look-ahead (mloam_frame_set_next*), so that the branch
//                           undistorts, merges and down-samples it too
//   k_undistort             TransformToEnd of the less-sharp and less-flat features of every LiDAR, in the LiDAR's frame, between the
//                           extraction and the rig merge (the reference undistorts cur_feature_ before the mapper sees it; the sharp and
//                           flat clouds and the outlier cloud are left as they are, and so is what the tracker kept in prev_feature_)
#include <cmath>
#include <cstring>

#include "ctx.h"
#include "host_util.h"

namespace mloam {

namespace {

// One thread per point of the two clouds: [0, cap_less) less-sharp, [cap_less, cap_less + cap_flat) less-flat
__global__ void __launch_bounds__(256) k_undistort(float4 *__restrict__ less_sharp, int cap_less, const int *__restrict__ n_less,
                                                   float4 *__restrict__ less_flat, int cap_flat, const int *__restrict__ n_flat,
                                                   const int *__restrict__ off, int n_lidars, const UndistStage *__restrict__ cfg) {
  const int g = blockIdx.x * blockDim.x + threadIdx.x;
  const bool flat = g >= cap_less;
  const int i = flat ? g - cap_less : g;
  if (i >= min(flat ? cap_flat : cap_less, flat ? *n_flat : *n_less)) return;
  float4 *pts = flat ? less_flat : less_sharp;
  int l = 0;
  if (off) {  // the rig's per-LiDAR offsets of this cloud (lidar_offsets_device), as k_merge_transform finds a point's LiDAR
    const int *o = flat ? off + n_lidars + 1 : off;
    while (l + 1 < n_lidars && i >= o[l + 1]) l++;
  }
  const float4 q = pts[i];
  float p[4] = {q.x, q.y, q.z, q.w};
  ud::transform_to_end(cfg->pose[l], cfg->scan_period, p, ud::sin_fd);
  pts[i] = make_float4(p[0], p[1], p[2], q.w);
}

// Pose::inverse (pose.cpp:99-102): Pose(q.inverse(), -(q.inverse() * t)), q.inverse() = conj(q) / squaredNorm(q), the Pose normalising
// its quaternion; q of a Pose is normalised already
PoseD pose_inverse_exact(const PoseD &a) {
  const double n2 = a.q.x * a.q.x + a.q.y * a.q.y + a.q.z * a.q.z + a.q.w * a.q.w;
  const Q4 qi{-a.q.x / n2, -a.q.y / n2, -a.q.z / n2, a.q.w / n2};
  return PoseD{qnormalized(qi), neg(qrot(qi, a.t))};
}
// Pose::operator* (pose.cpp:110-113): Pose(q1 q2, q1 t2 + t1), normalised
PoseD pose_mul(const PoseD &a, const PoseD &b) { return PoseD{qnormalized(qmul(a.q, b.q)), qrot(a.q, b.t) + a.t}; }

}  // namespace

namespace {
void stage_poses(Ctx *c, int n, const double (*pose7)[7], UndistStage *u) {
  memset(u, 0, sizeof(*u));
  u->scan_period = c->cfg.undist_scan_period, u->n_lidars = n;
  for (int l = 0; l < n; l++) ud::undist_pose_make(pose7[l], &u->pose[l]);
}
}  // namespace

void stage_undistort(Ctx *c, int parity, const UndistPoses *ahead) {
  stage_poses(c, c->undist_n, c->undist_pose7, &c->pinned->undist[parity]);
  if (ahead) stage_poses(c, ahead->n, ahead->pose7, &c->pinned->undist[parity ^ 1]);
}

void undist_withdraw(Ctx *c) {
  c->next.undist_open = false, c->next.undist.n = 0;
  c->undist_announced.undist.n = 0;
  if (c->prefetched.undist.n) c->prefetched.valid = false;
}

int undistort_stage(Ctx *c, int parity, ExtractOut out, int cap_less, int cap_flat, const int *d_off, int n_lidars) {
  UndistStage *d_cfg = nullptr;
  MLOAM_CUDA_OK(c, carve(c->undist, [&](Carve &cv) { d_cfg = cv.take<UndistStage>(2) + parity; }));
  ProfScope ps(c, "undistort");
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_cfg, &c->pinned->undist[parity], sizeof(UndistStage), cudaMemcpyHostToDevice, st));
  const long long total = (long long)cap_less + cap_flat;
  if (total <= 0) return MLOAM_OK;
  k_undistort<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(out.less_sharp, cap_less, out.counts + 1, out.less_flat, cap_flat, out.counts + 3,
                                                                d_off, n_lidars, d_cfg);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_undistort_poses(const double *pose_rlt7, int idx_ref, int n_lidars, const double *ext7s, int estimate_extrinsic, double *out7s) {
  if (!pose_rlt7 || !ext7s || !out7s || n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS || idx_ref < 0 || idx_ref >= n_lidars)
    return MLOAM_E_INVALID;
  const PoseD rlt = pose_from_param(pose_rlt7);  // as the odometry's Pose holds it (unit quaternion), not normalised again
  PoseD und[MLOAM_MAX_LIDARS];
  for (int n = 0; n < n_lidars; n++) {
    const double *e = ext7s + 7 * n;
    const PoseD ext{qnormalized(Q4{e[3], e[4], e[5], e[6]}), D3{e[0], e[1], e[2]}};  // Pose(qbl_[n], tbl_[n])
    und[n] = pose_mul(pose_mul(pose_inverse_exact(ext), rlt), ext);
  }
  for (int n = 0; n < n_lidars; n++) {
    const PoseD &p = und[estimate_extrinsic == 2 ? n : idx_ref];
    double *o = out7s + 7 * n;
    o[0] = p.t.x, o[1] = p.t.y, o[2] = p.t.z, o[3] = p.q.x, o[4] = p.q.y, o[5] = p.q.z, o[6] = p.q.w;
  }
  return MLOAM_OK;
}

int mloam_set_distortion(mloam_ctx_t *h, int on, float scan_period) {
  if (!h || (on != 0 && on != 1) || (on && !(scan_period > 0.f && scan_period <= 3.0e38f))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (multi_gpu(c))
    return fail(c, MLOAM_E_STATE, "set_distortion: the undistortion is single-GPU only, like with_ua; detach the communicator");
  c->cfg.undist_on = on != 0;
  if (on) c->cfg.undist_scan_period = scan_period;
  c->undist_set = false;
  undist_withdraw(c);
  return MLOAM_OK;
}

int mloam_frame_undistort(mloam_ctx_t *h, int n_lidars, const double *pose7) {
  if (!h || !pose7 || n_lidars < 1 || n_lidars > MLOAM_MAX_LIDARS) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->cfg.undist_on) return fail(c, MLOAM_E_STATE, "frame_undistort: turn the undistortion on first (mloam_set_distortion)");
  for (int k = 0; k < 7 * n_lidars; k++)
    if (!std::isfinite(pose7[k])) return fail(c, MLOAM_E_INVALID, "frame_undistort: non-finite pose");
  memcpy(c->undist_pose7, pose7, sizeof(double) * 7 * (size_t)n_lidars);
  c->undist_n = n_lidars, c->undist_set = true;
  return MLOAM_OK;
}

int mloam_frame_set_next_undistort(mloam_ctx_t *h, int n_lidars, const double *pose7) {
  if (!h || !pose7) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (!c->cfg.undist_on) return fail(c, MLOAM_E_STATE, "frame_set_next_undistort: turn the undistortion on first (mloam_set_distortion)");
  if (!c->next.set) return fail(c, MLOAM_E_STATE, "frame_set_next_undistort: no sweep is announced (mloam_frame_set_next*)");
  if (!c->next.undist_open)
    return fail(c, MLOAM_E_STATE, "frame_set_next_undistort: a setter withdrew the announcement's poses since the sweep was announced; "
                                  "announce it again (mloam_frame_set_next*)");
  if (multi_gpu(c))
    return fail(c, MLOAM_E_STATE, "frame_set_next_undistort: the undistortion is single-GPU only; detach the communicator");
  if (n_lidars != c->cfg.n_parts())
    return fail(c, MLOAM_E_INVALID, "frame_set_next_undistort: a pose count other than the frame's LiDARs (1 without the rig merge)");
  for (int k = 0; k < 7 * n_lidars; k++)
    if (!std::isfinite(pose7[k])) return fail(c, MLOAM_E_INVALID, "frame_set_next_undistort: non-finite pose");
  memcpy(c->next.undist.pose7, pose7, sizeof(double) * 7 * (size_t)n_lidars);
  c->next.undist.n = n_lidars;
  return MLOAM_OK;
}

}  // extern "C"
