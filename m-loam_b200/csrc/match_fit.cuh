// match_fit.cuh — the line / plane fit of one feature from its K neighbour positions (the second half of match*FromMap:
// feature_extract.hpp:410-458, 573-618, 670-715, 817-861).  One THREAD per feature; used by k_match_fit (match_kernels.cu) and,
// when the caller defers the fit, by the first evaluation of a solve (k_linearize, solve_kernels.cu) — the fit depends on the
// neighbour list only, so it can run in the thread that evaluates the feature's residual right afterwards.
#pragma once
#include "ctx.h"
#include "fit.cuh"

namespace mloam {

// FOV gate, feature_extract.hpp:696-715 (and :434-458, :599-618, :842-861)
__device__ __forceinline__ bool in_laser_fov(const PoseD &T, const float3 &sel) {
  const float3 zt = associate(T, 0.0f, 0.0f, 10.0f);
  const double ex = T.t.x - (double)sel.x, ey = T.t.y - (double)sel.y, ez = T.t.z - (double)sel.z;
  const float s1 = (float)(ex * ex + ey * ey + ez * ez);
  const float ax = zt.x - sel.x, ay = zt.y - sel.y, az = zt.z - sel.z;
  const float s2 = ax * ax + ay * ay + az * az;
  const float check1 = 100.0f + s1 - s2 - 10.0f * sqrtf(3.0f) * sqrtf(s1);
  const float check2 = 100.0f + s1 - s2 + 10.0f * sqrtf(3.0f) * sqrtf(s1);
  return check1 < 0 && check2 > 0;
}


// Returns whether it fitted (false: the list is unchanged and valid / coeff stand).  ok_out / coeff_out (nullable) receive what it
// stores, so that a caller that evaluates the feature next need not read it back.
template <int K>
__device__ __forceinline__ bool fit_one(const FitSet &s, int j, const PoseD &T, float min_plane_dis, int check_fov, bool *ok_out = nullptr,
                                        float *coeff_out = nullptr) {
  // The fit depends on the map points only: with an unchanged neighbour list the previous iteration's valid / coeff
  // stand (the FOV gate depends on the pose, so it disables the shortcut).
  if (s.changed && !check_fov && !s.changed[j]) return false;
  const int *ps = s.pos + (size_t)j * K;
  bool ok = ps[0] >= 0;
  float out[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
  int idx[K];
#pragma unroll
  for (int k = 0; k < K; k++) idx[k] = -1;
  if (ok) {
    float X[K][3];
#pragma unroll
    for (int k = 0; k < K; k++) {
      const float4 v = __ldg(s.sorted + ps[k]);
      X[k][0] = v.x, X[k][1] = v.y, X[k][2] = v.z;
      idx[k] = __float_as_int(v.w);
    }
    if (s.is_plane) {
      // :573-594 / :817-837
      float A[K][3];
#pragma unroll
      for (int k = 0; k < K; k++) A[k][0] = X[k][0], A[k][1] = X[k][1], A[k][2] = X[k][2];
      float nv[3];
      ok = lsq_plane_dev<K>(A, nv);
      if (ok) {
        const float nrm = sqrtf(nv[0] * nv[0] + nv[1] * nv[1] + nv[2] * nv[2]);
        const float d = 1 / nrm;
        nv[0] = nv[0] / nrm, nv[1] = nv[1] / nrm, nv[2] = nv[2] / nrm;
#pragma unroll
        for (int k = 0; k < K; k++)
          if (fabsf(nv[0] * X[k][0] + nv[1] * X[k][1] + nv[2] * X[k][2] + d) > min_plane_dis) ok = false;
        out[0] = nv[0], out[1] = nv[1], out[2] = nv[2], out[3] = d;
      }
    } else {
      // :410-432 / :670-693
      float cx = 0.f, cy = 0.f, cz = 0.f;
#pragma unroll
      for (int k = 0; k < K; k++) cx = cx + X[k][0], cy = cy + X[k][1], cz = cz + X[k][2];
      const float kf = (float)K;
      cx = cx / kf, cy = cy / kf, cz = cz / kf;
      float c00 = 0.f, c01 = 0.f, c02 = 0.f, c11 = 0.f, c12 = 0.f, c22 = 0.f;
#pragma unroll
      for (int k = 0; k < K; k++) {
        const float a = X[k][0] - cx, b = X[k][1] - cy, c = X[k][2] - cz;
        c00 = c00 + a * a, c01 = c01 + a * b, c02 = c02 + a * c;
        c11 = c11 + b * b, c12 = c12 + b * c, c22 = c22 + c * c;
      }
      float w[3], V[3][3];
      eig3f_dev(c00, c01, c02, c11, c12, c22, w, V);
      ok = w[2] > 3 * w[1];
      const float k01 = 0.1f;
      out[0] = k01 * V[0][2] + cx, out[1] = k01 * V[1][2] + cy, out[2] = k01 * V[2][2] + cz;
      out[3] = -k01 * V[0][2] + cx, out[4] = -k01 * V[1][2] + cy, out[5] = -k01 * V[2][2] + cz;
    }
    if (ok && check_fov) {
      const float4 p = __ldg(s.pts + j);
      ok = in_laser_fov(T, associate(T, p.x, p.y, p.z));
    }
  }
  s.valid[j] = ok ? 1 : 0;
#pragma unroll
  for (int k = 0; k < 6; k++) s.coeff[(size_t)j * 6 + k] = ok ? out[k] : 0.f;
  if (s.nn) {
#pragma unroll
    for (int k = 0; k < K; k++) s.nn[(size_t)j * K + k] = ok ? idx[k] : -1;
  }
  if (ok_out) {
    *ok_out = ok;
#pragma unroll
    for (int k = 0; k < 6; k++) coeff_out[k] = ok ? out[k] : 0.f;
  }
  return true;
}


}  // namespace mloam
