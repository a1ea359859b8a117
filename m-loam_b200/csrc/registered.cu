// registered.cu — pubPointCloud (lidar_mapper_keyframe.cpp:690-714) in the frame path: the three clouds the mapper publishes every frame,
// moved into the world frame with the optimised pose pose_wmap_curr:
//   MLOAM_REGISTERED_FULL_RES  laser_cloud_full_res += laser_cloud_outlier (:693-699): the ring-ordered sweep LiDAR by LiDAR — each point
//                              [TransformToEnd with the LiDAR's pose_undist, estimator.cpp:405] -> the base frame as the frame moves its
//                              less-* features (transformCloudFeature with intensity = l, visualization.cpp:40-52, every point: the
//                              cloud is dense for PCL; or pointAssociateToMap with the single extrinsic; or nothing) — then, with the
//                              outlier cloud on, its pre-filter input (one point per LiDAR, not undistorted)
//   MLOAM_REGISTERED_SURF      laser_cloud_surf_last (:701-706): the merged surf_points_less_flat before downsampleCurrentScan's filter
//   MLOAM_REGISTERED_CORNER    laser_cloud_corner_last (:708-713): the same for corner_points_less_sharp
// and pointAssociateToMap(., pose_wmap_curr) (utility.h:103-117) on every point.  One launch: k_registered.
#include <algorithm>
#include <cstring>

#include "ctx.h"
#include "host_util.h"

namespace mloam {

namespace {

constexpr int REG_THREADS = 256;

// Grid-stride over the points of the three clouds, in output order: the sweep's n_sweep points, MLOAM_MAX_LIDARS outlier slots, the
// less-flat then the less-sharp features.  Every block reads the counts; block 0 publishes them.
__global__ void __launch_bounds__(REG_THREADS) k_registered(const RegArgs a, const RegOut o) {
  __shared__ double s_pose[7];
  __shared__ int s_start[MLOAM_MAX_LIDARS];
  __shared__ int s_n[4];  // sweep, outlier points, less-flat, less-sharp
  const int tid = threadIdx.x;
  if (tid < 7) s_pose[tid] = a.pose[tid];
  if (tid < a.n_parts) s_start[tid] = a.scan_start[tid * a.rings_per_lidar] - 5;  // LiDAR l's part of the sweep (prepare_multi's cut)
  if (tid == 0) {
    s_n[0] = a.d_n_sweep ? min(a.n_sweep, *a.d_n_sweep) : a.n_sweep;
    int k = 0;
    if (a.first)
      for (int l = 0; l < a.n_parts; l++) k += a.first_ok[l] ? 1 : 0;
    s_n[1] = k;
    s_n[2] = min(a.cap_flat, *a.n_flat), s_n[3] = min(a.cap_sharp, *a.n_sharp);
    if (blockIdx.x == 0) o.counts[0] = s_n[0] + s_n[1], o.counts[1] = s_n[2], o.counts[2] = s_n[3];
  }
  __syncthreads();
  const PoseD T = pose_from_param(s_pose);
  const int ns = s_n[0], nf = s_n[2], nc = s_n[3];
  const long long b1 = ns, b2 = b1 + MLOAM_MAX_LIDARS, b3 = b2 + nf, total = b3 + nc;
  for (long long g = (long long)blockIdx.x * REG_THREADS + tid; g < total; g += (long long)gridDim.x * REG_THREADS) {
    float4 p;
    float4 *dst;
    if (g < b1) {  // the sweep: [undistortion] -> base frame
      const int i = (int)g;
      int l = 0;
      while (l + 1 < a.n_parts && i >= s_start[l + 1]) l++;
      const float4 r = a.sweep[i];
      float q[4] = {r.x, r.y, r.z, r.w};
      if (a.undist) ud::transform_to_end(a.undist->pose[l], a.undist->scan_period, q, ud::sin_fd);  // as k_undistort
      p = make_float4(q[0], q[1], q[2], r.w);
      if (a.to_base == 1) {
        p = rig_transform(a.rig + 12 * l, p, (float)l);  // as k_merge_transform
      } else if (a.to_base == 2) {
        const float3 e = associate(pose_from_param(a.ext), p.x, p.y, p.z);  // as k_transform_points
        p = make_float4(e.x, e.y, e.z, p.w);
      }
      dst = o.cloud[0] + i;
    } else if (g < b2) {  // laser_cloud_outlier: LiDAR l's first point, if its part is not empty, as k_outlier_scan takes it
      const int l = (int)(g - b1);
      if (!a.first || l >= a.n_parts || !a.first_ok[l]) continue;
      int at = 0;
      for (int k = 0; k < l; k++) at += a.first_ok[k] ? 1 : 0;
      p = rig_transform(a.outlier->mat[l], a.first[l], (float)l);
      dst = o.cloud[0] + ns + at;
    } else if (g < b3) {
      const int i = (int)(g - b2);
      p = a.less_flat[i];
      dst = o.cloud[1] + i;
    } else {
      const int i = (int)(g - b3);
      p = a.less_sharp[i];
      dst = o.cloud[2] + i;
    }
    const float3 w = associate(T, p.x, p.y, p.z);  // pointAssociateToMap(., pose_wmap_curr), intensity kept
    *dst = make_float4(w.x, w.y, w.z, p.w);
  }
}

}  // namespace

int registered_layout(Ctx *c, int n_sweep, int cap_flat, int cap_sharp, RegOut *o) {
  o->cap[0] = n_sweep + MLOAM_MAX_LIDARS, o->cap[1] = cap_flat, o->cap[2] = cap_sharp;
  MLOAM_CUDA_OK(c, carve(c->registered, [&](Carve &cv) {
    for (int t = 0; t < 3; t++) o->cloud[t] = cv.take<float4>((size_t)o->cap[t] + 1);
    o->counts = cv.take<int>(4);
  }));
  return MLOAM_OK;
}

int registered_stage(Ctx *c, const RegArgs &a, const RegOut &o) {
  if (a.n_parts < 1 || a.n_parts > MLOAM_MAX_LIDARS || a.rings_per_lidar < 1) return fail(c, MLOAM_E_INVALID, "registered: 1..16 LiDARs");
  ProfScope ps(c, "registered");
  const long long work = (long long)a.n_sweep + MLOAM_MAX_LIDARS + a.cap_flat + a.cap_sharp;
  const long long grid = std::min<long long>((work + REG_THREADS - 1) / REG_THREADS, 8ll * c->sm_count);
  k_registered<<<(unsigned)grid, REG_THREADS, 0, c->stream>>>(a, o);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

namespace {

// The checks both read-backs make; *m = the cloud's size
int registered_count(Ctx *c, int which, int *m) {
  *m = 0;
  if (which < MLOAM_REGISTERED_FULL_RES || which > MLOAM_REGISTERED_CORNER)
    return fail(c, MLOAM_E_INVALID, "frame_registered: which must be MLOAM_REGISTERED_FULL_RES, _SURF or _CORNER");
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "frame_registered: the registered clouds are single-GPU only; detach the communicator");
  if (!c->reg_valid)
    return fail(c, MLOAM_E_STATE, "frame_registered: the last call was no mloam_frame* call run with the registered clouds on (mloam_set_registered)");
  cudaSetDevice(c->device);
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, c->reg_last.counts + which, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  *m = hc[0];
  return MLOAM_OK;
}

}  // namespace

extern "C" {

int mloam_set_registered(mloam_ctx_t *h, int on) {
  if (!h || (on != 0 && on != 1)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (on && multi_gpu(c))
    return fail(c, MLOAM_E_STATE, "set_registered: the registered clouds are single-GPU only, like with_ua; detach the communicator");
  c->cfg.reg_on = on != 0;
  return MLOAM_OK;
}

int mloam_frame_registered(mloam_ctx_t *h, int which, mloam_point_t *h_pts, int cap, int *n) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (n) *n = 0;
  int m = 0;
  const int rc = registered_count(c, which, &m);
  if (rc) return rc;
  if (n) *n = m;
  if (!h_pts || m == 0) return MLOAM_OK;
  if (m > cap) return fail(c, MLOAM_E_INVALID, "frame_registered: capacity too small (*n holds the cloud's size)");
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_pts, c->reg_last.cloud[which], sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  return MLOAM_OK;
}

int mloam_frame_registered_device(mloam_ctx_t *h, int which, const mloam_point_t **d_pts, int *n) {
  if (!h || !d_pts || !n) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  *d_pts = nullptr, *n = 0;
  int m = 0;
  const int rc = registered_count(c, which, &m);
  if (rc) return rc;
  *d_pts = reinterpret_cast<const mloam_point_t *>(c->reg_last.cloud[which]), *n = m;
  return MLOAM_OK;
}

}  // extern "C"
