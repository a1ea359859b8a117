// host_util.h — small host-side helpers shared by the C-ABI translation units.
#pragma once
#include <cmath>
#include <cstring>
#include "ctx.h"

namespace mloam {

inline int fail(Ctx *c, int code, const char *msg) {
  c->err = msg;
  return code;
}

inline MatchCfg match_cfg(const Ctx *c) {
  MatchCfg m;
  m.min_match_sq_dis = c->params.min_match_sq_dis;
  m.min_plane_dis = c->params.min_plane_dis;
  m.n_neigh = c->params.n_neigh;
  m.check_fov = c->params.check_fov;
  return m;
}

inline double map_sqrt_info(double cov_trace) {  // lidar_map_factor.hpp:34,41
  double s = sqrt(1 / cov_trace);
  return s >= 3.0 ? 1.0 : s / 3.0;
}

inline float pick_cell(const Ctx *c, float requested) {
  // <= 0: map_build_device picks the slot's sticky auto cell (ctx.h MapStorage::auto_cell_pick)
  float cell = requested > 0.f ? requested : (c->params.map_cell > 0.f ? c->params.map_cell : 0.f);
  return cell;
}

// Pose(q, t).T_.cast<float>() of the pose e7 (pose.cpp:34-41): q normalised, [R | t] row-major as a float 3x4
inline void pose_mat12(const double *e7, float *m12) {
  const M33 R = qmat(qnormalized(Q4{e7[3], e7[4], e7[5], e7[6]}));
  for (int r = 0; r < 3; r++) {
    for (int k = 0; k < 3; k++) m12[4 * r + k] = (float)R.m[3 * r + k];
    m12[4 * r + 3] = (float)e7[r];
  }
}

inline int upload_pose(Ctx *c, const double *pose7, double **d_pose) {
  double *stage = c->pinned->upload_pose;
  for (int k = 0; k < 7; k++) stage[k] = pose7[k];
  double *d = c->ctl.as<DevCtl>()->upload_pose;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d, stage, 7 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  *d_pose = d;
  return MLOAM_OK;
}

inline int reserve_feat(Ctx *c, int t, int n) {
  MLOAM_CUDA_OK(c, c->feat_valid[t].reserve((size_t)n + 16));
  MLOAM_CUDA_OK(c, c->feat_coeff[t].reserve(sizeof(float) * 6 * (size_t)(n + 1)));
  MLOAM_CUDA_OK(c, c->feat_nn[t].reserve(sizeof(int) * (size_t)c->params.n_neigh * (size_t)(n + 1)));
  return MLOAM_OK;
}


}  // namespace mloam
