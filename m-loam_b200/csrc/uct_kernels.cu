// uct_kernels.cu — uncertainty-aware mapping inputs (SURVEY.md §8 row a24).
//   k_point_uncertainty  evalPointUncertainty (estimator/src/lidarMapper/associate_uct.hpp:164-215, pointToFS :149-156):
//                        cov_point = top-left 3x3 of G diag(cov_pose, COV_MEASUREMENT) G^T with G = [I3 | -[T p]x | R],
//                        one thread per point, stored like PointIWithCov::cov_vec (float [xx xy xz yy yz zz]).
//   k_sqrt_info          extractCov -> trace -> sqrt(1/trace) with the clamp of lidar_map_factor.hpp:34,41, one
//                        double per scan point, consumed by k_linearize (with_ua = true, lidar_mapper_keyframe.cpp:541-560).
#include "ctx.h"
#include "host_util.h"

namespace mloam {

struct UctArgs {
  double pose[7];
  double cov_pose[36];
  double cov_meas[9];
};

__global__ void k_point_uncertainty(const float4 *__restrict__ pts, int n, UctArgs a, float *__restrict__ cov6) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const float4 p = pts[i];
  const PoseD T = pose_from_param(a.pose);
  const D3 tp = qrot(T.q, D3{(double)p.x, (double)p.y, (double)p.z}) + T.t;
  const M33 R = qmat(T.q);
  // rows of G (3 x 9): [e_i | -([tp]x)_i | R_i]
  double G[3][9];
  const double S[9] = {0.0, -tp.z, tp.y, tp.z, 0.0, -tp.x, -tp.y, tp.x, 0.0};
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = 0; c < 3; c++) G[r][c] = (r == c) ? 1.0 : 0.0, G[r][3 + c] = -S[r * 3 + c], G[r][6 + c] = R.m[r * 3 + c];
  double C[6];
  int q = 0;
#pragma unroll
  for (int r = 0; r < 3; r++)
#pragma unroll
    for (int c = r; c < 3; c++) {
      double s = 0;
      for (int u = 0; u < 9; u++) {
        double t = 0;
        for (int v = 0; v < 9; v++) {
          const double sig = (u < 6 && v < 6) ? a.cov_pose[u * 6 + v] : ((u >= 6 && v >= 6) ? a.cov_meas[(u - 6) * 3 + (v - 6)] : 0.0);
          t += sig * G[c][v];
        }
        s += G[r][u] * t;
      }
      C[q++] = s;
    }
#pragma unroll
  for (int k = 0; k < 6; k++) cov6[(size_t)i * 6 + k] = (float)C[k];
}

__global__ void k_sqrt_info(const float *__restrict__ cov6, int n, double *__restrict__ sinfo) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  sinfo[i] = cov6_sqrt_info(cov6 + (size_t)i * 6);
}

int sqrt_info_device(Ctx *c, const float *d_cov6, int n, double *d_sinfo) {
  if (n <= 0) return MLOAM_OK;
  k_sqrt_info<<<(n + 255) / 256, 256, 0, c->stream>>>(d_cov6, n, d_sinfo);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

extern "C" int mloam_point_uncertainty(mloam_ctx_t *h, const mloam_point_t *h_pts, int n, const double *pose7, const double *cov_pose36,
                                       const double *cov_meas9, float *h_cov6) {
  if (!h || n < 0 || !pose7 || !cov_pose36 || !cov_meas9 || (n > 0 && (!h_pts || !h_cov6))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (n == 0) return MLOAM_OK;
  MLOAM_CUDA_OK(c, c->sweep_in.reserve(sizeof(float4) * (size_t)n));
  MLOAM_CUDA_OK(c, c->map_in[0].reserve(sizeof(float) * 6 * (size_t)n));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->sweep_in.p, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, c->stream));
  UctArgs a;
  memcpy(a.pose, pose7, sizeof(a.pose));
  memcpy(a.cov_pose, cov_pose36, sizeof(a.cov_pose));
  memcpy(a.cov_meas, cov_meas9, sizeof(a.cov_meas));
  k_point_uncertainty<<<(n + 127) / 128, 128, 0, c->stream>>>(c->sweep_in.as<float4>(), n, a, c->map_in[0].as<float>());
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6, c->map_in[0].p, sizeof(float) * 6 * (size_t)n, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}
