// submap.cu — submap assembly with uncertainty (SURVEY.md 8f item 2): the data path of extractSurroundingKeyFrames
// (lidar_mapper_keyframe.cpp:254-354) on the device, so that the submap is BUILT where it is searched:
//
//   mloam_compound_pose_cov      compoundPoseWithCov (associate_uct.hpp:9-88, method 2) — host-side 6x6 algebra, once per keyframe / LiDAR
//   k_uct_associate              cloudUCTAssociateToMap (:1116-1158): per point  ext^-1 -> evalPointUncertainty under the compound
//                                pose (trace gate) -> pointAssociateToMap with the keyframe pose -> updateCov; stable compaction
//   voxel_downsample_cov_device  VoxelGridCovarianceMLOAM<PointIWithCov> with the covariance-weighted merge (extract_kernels.cu)
//   mloam_submap_assemble        all surrounding keyframes of one map -> merged cloud -> filter -> map slot (setInputCloud), no host copy
//                                of the points in between
#include <vector>

#include "ctx.h"
#include "host_util.h"
#include "uct.h"

namespace mloam {

// One point of cloudUCTAssociateToMap: its associated point, cov_vec and trace at index i of out / cov6 / trace, and whether it passes
// the trace gate.  pose_global: f.pose_global, or the keyframe pose of a batched run (k_uct_associate_seg).
__device__ __forceinline__ int uct_point(const float4 po, const UctFrame &f, const double *pose_global, const UctLaser *__restrict__ lasers,
                                         size_t i, float4 *__restrict__ out, float *__restrict__ cov6, float *__restrict__ trace) {
  int ind = (int)po.w;  // laser id in the intensity (:1143)
  ind = ind < 0 ? 0 : (ind >= f.n_lasers ? f.n_lasers - 1 : ind);
  double C[6] = {0, 0, 0, 0, 0, 0};
  int ok = 1;
  if (f.with_ua) {
    const UctLaser &L = lasers[ind];
    const float3 sel = associate(pose_from_param(L.ext_inv), po.x, po.y, po.z);  // :1147
    // evalPointUncertainty (associate_uct.hpp:192-214) under the compound pose: G = [I3 | -[T p]x | R], Sigma = diag(cov_pose, COV_MEASUREMENT)
    const PoseD T = pose_from_param(L.compound);
    const D3 tp = qrot(T.q, D3{(double)sel.x, (double)sel.y, (double)sel.z}) + T.t;
    const M33 R = qmat(T.q);
    double G[3][9];
    const double S[9] = {0.0, -tp.z, tp.y, tp.z, 0.0, -tp.x, -tp.y, tp.x, 0.0};
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = 0; c < 3; c++) G[r][c] = (r == c) ? 1.0 : 0.0, G[r][3 + c] = -S[r * 3 + c], G[r][6 + c] = R.m[r * 3 + c];
    int q = 0;
#pragma unroll
    for (int r = 0; r < 3; r++)
#pragma unroll
      for (int c = r; c < 3; c++) {
        double s = 0;
        for (int u = 0; u < 9; u++) {
          double t = 0;
          for (int v = 0; v < 9; v++) {
            const double sig = (u < 6 && v < 6) ? L.cov[u * 6 + v] : ((u >= 6 && v >= 6) ? f.cov_meas[(u - 6) * 3 + (v - 6)] : 0.0);
            t += sig * G[c][v];
          }
          s += G[r][u] * t;
        }
        C[q++] = s;
      }
    if (C[0] + C[3] + C[5] > f.trace_threshold) ok = 0;  // :1150
  }
  if (f.scan_frame) {
    out[i] = po;  // the scan stays in the base frame; only its covariance is attached (PointIWithCov(point_ori, cov), :385-386)
  } else {
    const float3 pc = associate(pose_from_param(pose_global), po.x, po.y, po.z);  // :1152
    out[i] = make_float4(pc.x, pc.y, pc.z, po.w);
  }
#pragma unroll
  for (int k = 0; k < 6; k++) cov6[i * 6 + k] = (float)C[k];  // updateCov (point_with_cov.hpp:187-196)
  trace[i] = (float)(C[0] + C[3] + C[5]);
  return ok;
}

// d_f (nullable): the frame read from device memory instead of `f` (staged by a captured H2D copy, so that a replay sees new values).
// d_n (nullable): device-side point count, n is then the launch bound; points beyond it are not kept.
__global__ void k_uct_associate(const float4 *__restrict__ pts, int n, UctFrame f, const UctLaser *__restrict__ lasers, float4 *__restrict__ out,
                                float *__restrict__ cov6, float *__restrict__ trace, int *__restrict__ keep, const UctFrame *__restrict__ d_f = nullptr,
                                const int *__restrict__ d_n = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  if (d_n && i >= *d_n) {
    keep[i] = 0;
    return;
  }
  if (d_f) f = *d_f;
  keep[i] = uct_point(pts[i], f, f.pose_global, lasers, (size_t)i, out, cov6, trace);
}

// The association of many keyframe clouds in one launch: point i of the concatenated input belongs to the last segment whose begin is
// <= i (segments are non-empty and in output order); it is read straight from the keyframe's record and associated with that keyframe's
// pose (kf_pose7[7 * kf]) and UctLaser block (lasers[f.n_lasers * kf]).
__global__ void k_uct_associate_seg(const UctSeg *__restrict__ seg, int n_seg, int n, UctFrame f, const double *__restrict__ kf_pose7,
                                    const UctLaser *__restrict__ lasers, float4 *__restrict__ out, float *__restrict__ cov6,
                                    float *__restrict__ trace, int *__restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  int lo = 0, hi = n_seg - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (seg[mid].begin <= i) lo = mid;
    else hi = mid - 1;
  }
  const UctSeg s = seg[lo];
  keep[i] = uct_point(s.pts[i - s.begin], f, kf_pose7 + 7 * (size_t)s.kf, lasers + (size_t)f.n_lasers * s.kf, (size_t)i, out, cov6, trace);
}

__global__ void k_compact_cov(const float4 *__restrict__ pts, const float *__restrict__ cov6, const float *__restrict__ trace, const int *__restrict__ keep,
                              const int *__restrict__ slot, int n, int dst_off, const int *__restrict__ d_dst_off, float4 *__restrict__ out,
                              float *__restrict__ cov6_out, float *__restrict__ trace_out, double *__restrict__ sinfo_out = nullptr) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n || !keep[i]) return;
  const int o = (d_dst_off ? *d_dst_off : dst_off) + slot[i];
  out[o] = pts[i];
#pragma unroll
  for (int k = 0; k < 6; k++) cov6_out[(size_t)o * 6 + k] = cov6[(size_t)i * 6 + k];
  trace_out[o] = trace[i];
  if (sinfo_out) sinfo_out[o] = cov6_sqrt_info(cov6 + (size_t)i * 6);  // the factor's weight (extractCov + lidar_map_factor.hpp:34,41)
}
__global__ void k_add_count(int *total, const int *part) {
  if (threadIdx.x == 0 && blockIdx.x == 0) *total += *part;
}

// host-side 3x3 / 6x6 helpers for compoundPoseWithCov
namespace {
struct H3 {
  double m[9];
};
struct H6 {
  double m[36];
};
H3 h3_mul(const H3 &A, const H3 &B) {
  H3 C;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) C.m[i * 3 + j] = A.m[i * 3] * B.m[j] + A.m[i * 3 + 1] * B.m[3 + j] + A.m[i * 3 + 2] * B.m[6 + j];
  return C;
}
H3 h3_add(const H3 &A, const H3 &B) {
  H3 C;
  for (int i = 0; i < 9; i++) C.m[i] = A.m[i] + B.m[i];
  return C;
}
H3 h3_T(const H3 &A) {
  H3 T;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) T.m[i * 3 + j] = A.m[j * 3 + i];
  return T;
}
H3 covop1(const H3 &B) {  // associate_uct.hpp:18-22
  const double tr = B.m[0] + B.m[4] + B.m[8];
  H3 A = B;
  for (int i = 0; i < 3; i++) A.m[i * 4] = -tr + B.m[i * 4];
  return A;
}
H3 covop2(const H3 &B, const H3 &C) { return h3_add(h3_mul(covop1(B), covop1(C)), covop1(h3_mul(C, B))); }  // :24-28
H6 h6_mul(const H6 &A, const H6 &B) {
  H6 C;
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) {
      double s = 0;
      for (int k = 0; k < 6; k++) s += A.m[i * 6 + k] * B.m[k * 6 + j];
      C.m[i * 6 + j] = s;
    }
  return C;
}
H6 h6_T(const H6 &A) {
  H6 T;
  for (int i = 0; i < 6; i++)
    for (int j = 0; j < 6; j++) T.m[i * 6 + j] = A.m[j * 6 + i];
  return T;
}
H3 blk(const H6 &A, int r0, int c0) {
  H3 B;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) B.m[i * 3 + j] = A.m[(r0 + i) * 6 + c0 + j];
  return B;
}
void put(H6 &A, int r0, int c0, const H3 &B) {
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) A.m[(r0 + i) * 6 + c0 + j] = B.m[i * 3 + j];
}
void pose_inverse(const double *x, double *out) {  // Pose::inverse (pose.cpp:99-102): conj(q), -(conj(q) * t); q normalised (Pose ctor)
  const Q4 qi = qnormalized(qconj(Q4{x[3], x[4], x[5], x[6]}));
  const D3 t = neg(qrot(qi, D3{x[0], x[1], x[2]}));
  out[0] = t.x, out[1] = t.y, out[2] = t.z, out[3] = qi.x, out[4] = qi.y, out[5] = qi.z, out[6] = qi.w;
}
}  // namespace

void uct_bufs_layout(Carve &cv, int n, UctBufs *B) {
  const size_t N1 = (size_t)n + 16;
  B->staged = cv.take<float4>(N1), B->cov6 = cv.take<float>(6 * N1), B->trace = cv.take<float>(N1);
  B->keep = cv.take<int>(N1), B->slot = cv.take<int>(N1), B->tmp = cv.take<int>(N1 / 2048 + 8), B->count = cv.take<int>(16);
}

int uct_bufs(Ctx *c, int n, UctBufs *B) {
  MLOAM_CUDA_OK(c, carve(c->assoc_work(), [&](Carve &cv) { uct_bufs_layout(cv, n, B); }));
  return MLOAM_OK;
}

int uct_associate_append(Ctx *c, const float4 *d_pts, int n, const UctFrame &f, const UctLaser *d_lasers, const UctBufs &B, float4 *d_out,
                                float *d_cov6_out, float *d_trace_out, int *d_total) {
  if (n <= 0) return MLOAM_OK;
  cudaStream_t st = c->stream;
  k_uct_associate<<<(n + 127) / 128, 128, 0, st>>>(d_pts, n, f, d_lasers, B.staged, B.cov6, B.trace, B.keep);
  scan_exclusive(c, B.keep, B.slot, n, B.tmp, B.count);
  k_compact_cov<<<(n + 255) / 256, 256, 0, st>>>(B.staged, B.cov6, B.trace, B.keep, B.slot, n, 0, d_total, d_out, d_cov6_out, d_trace_out);
  k_add_count<<<1, 32, 0, st>>>(d_total, B.count);
  c->launches += 3;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

int uct_associate_segments(Ctx *c, const UctSeg *d_seg, int n_seg, int n, const UctFrame &f, const double *d_kf_pose7, const UctLaser *d_lasers,
                           const UctBufs &B, float4 *d_out, float *d_cov6_out, float *d_trace_out) {
  cudaStream_t st = c->stream;
  if (n <= 0 || n_seg <= 0) {
    MLOAM_CUDA_OK(c, cudaMemsetAsync(B.count, 0, sizeof(int), st));
    return MLOAM_OK;
  }
  k_uct_associate_seg<<<(n + 127) / 128, 128, 0, st>>>(d_seg, n_seg, n, f, d_kf_pose7, d_lasers, B.staged, B.cov6, B.trace, B.keep);
  c->launches++;
  scan_exclusive(c, B.keep, B.slot, n, B.tmp, B.count);
  k_compact_cov<<<(n + 255) / 256, 256, 0, st>>>(B.staged, B.cov6, B.trace, B.keep, B.slot, n, 0, nullptr, d_out, d_cov6_out, d_trace_out);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

void fill_lasers(int n_lasers, const double *ext7, const double *pose_compound7, const double *cov_compound36, std::vector<UctLaser> &L) {
  L.resize(n_lasers);
  for (int l = 0; l < n_lasers; l++) {
    pose_inverse(ext7 + 7 * l, L[l].ext_inv);
    for (int k = 0; k < 7; k++) L[l].compound[k] = pose_compound7[7 * l + k];
    for (int k = 0; k < 36; k++) L[l].cov[k] = cov_compound36[36 * l + k];
  }
}

// ---- the with_ua stage of a frame: downsampleCurrentScan's uncertainty loop (lidar_mapper_keyframe.cpp:376-407) for both scans.
// Per point, idx = int(intensity) (the laser id of the rig merge; 0 in the single-LiDAR path without it, where intensity still
// holds the ring): pointAssociateToMap with pose_ext[idx]^-1, evalPointUncertainty under pose_ext[idx] with its covariance, dropped
// when trace > TRACE_THRESHOLD_MAPPING; the kept points keep their order.  This is cloudUCTAssociateToMap's per-point work with the
// extrinsic as the compound pose and no pose_global transform, so k_uct_associate + k_compact_cov do it.
void ua_stage_host(Ctx *c) {
  UctFrame *f = &c->pinned->ua.frame;
  UctLaser *L = c->pinned->ua.lasers;
  const FrameCfg &cfg = c->cfg;
  const int n_lasers = cfg.n_parts();
  memset(f, 0, sizeof(*f));
  for (int k = 0; k < 7; k++) f->pose_global[k] = k == 6 ? 1.0 : 0.0;
  memcpy(f->cov_meas, cfg.ua_cov_meas, sizeof(f->cov_meas));
  f->trace_threshold = cfg.ua_trace_threshold, f->with_ua = 1, f->n_lasers = n_lasers, f->scan_frame = 1;
  for (int l = 0; l < n_lasers; l++) {
    // pose_ext[idx]: the extrinsic the features were moved to the base frame with (identity when there is none)
    const double *e = cfg.part_ext(l);
    pose_inverse(e, L[l].ext_inv);
    for (int k = 0; k < 7; k++) L[l].compound[k] = e[k];
    for (int k = 0; k < 36; k++) L[l].cov[k] = cfg.ua_ext_cov[l][k];
  }
}

int ua_scan_stage(Ctx *c, Ctx::ScanRef *S, const UaStage **d_cfg_out) {
  const int ncap[2] = {S->n_corner, S->n_surf};
  const float4 *pts[2] = {S->corner, S->surf};
  const int *d_n[2] = {S->d_n_corner, S->d_n_surf};
  // Ctx::ua_scan: the staged configuration, then per scan the association work and the gated scan
  UaStage *d_cfg = nullptr;
  UctBufs B[2];
  float4 *out[2];
  float *ocov6[2], *otrace[2];
  double *osinfo[2];
  MLOAM_CUDA_OK(c, carve(c->ua_scan, [&](Carve &cv) {
    d_cfg = cv.take<UaStage>(1);
    for (int t = 0; t < 2; t++) {
      const int n = ncap[t] > 0 ? ncap[t] : 0;
      const size_t N1 = (size_t)n + 16;
      uct_bufs_layout(cv, n, &B[t]);
      out[t] = cv.take<float4>(N1), ocov6[t] = cv.take<float>(6 * N1), otrace[t] = cv.take<float>(N1), osinfo[t] = cv.take<double>(N1);
    }
  }));
  if (d_cfg_out) *d_cfg_out = d_cfg;
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_cfg, &c->pinned->ua, sizeof(UaStage), cudaMemcpyHostToDevice, st));
  const UctFrame f_unused{};
  for (int t = 0; t < 2; t++) {
    const int n = ncap[t];
    const UctBufs &b = B[t];
    if (n > 0) {
      k_uct_associate<<<(n + 127) / 128, 128, 0, st>>>(pts[t], n, f_unused, d_cfg->lasers, b.staged, b.cov6, b.trace, b.keep, &d_cfg->frame, d_n[t]);
      c->launches++;
    }
    scan_exclusive(c, b.keep, b.slot, n, b.tmp, b.count);  // the gated count lands where the solve reads its feature count
    if (n > 0) {
      k_compact_cov<<<(n + 255) / 256, 256, 0, st>>>(b.staged, b.cov6, b.trace, b.keep, b.slot, n, 0, nullptr, out[t], ocov6[t], otrace[t], osinfo[t]);
      c->launches++;
    }
    MLOAM_CUDA_OK(c, cudaGetLastError());
    if (t == 0) S->corner = out[t], S->d_n_corner = b.count, S->sinfo_corner = osinfo[t], S->cov6_corner = ocov6[t];
    else S->surf = out[t], S->d_n_surf = b.count, S->sinfo_surf = osinfo[t], S->cov6_surf = ocov6[t];
  }
  return MLOAM_OK;
}

// ---- the outlier cloud of a frame with segment_cloud: 0 (lidar_mapper_keyframe.cpp:366-418).  ImageSegmenter::segmentCloud pushes one
// point per LiDAR into laser_cloud_outlier, the first point of its ring-ordered cloud (image_segmenter.hpp:390; the extraction recorded
// it, ExtractOut::first), pubPointCloud moves it to the base frame with the float extrinsic, intensity = n (visualization.cpp:40-52,
// :89-104), and downsampleCurrentScan filters the merged cloud with VoxelGridCovarianceMLOAM<PointI>(MAP_OUTLIER_RES) (:366-368) and
// gates it as the scans (:407-418).  At most MLOAM_MAX_LIDARS points: one warp, the filter on lane 0.
void stage_outlier(Ctx *c) {
  OutlierStage *o = &c->pinned->outlier;
  memset(o, 0, sizeof(*o));
  o->leaf = c->cfg.outlier_leaf, o->n_lasers = c->cfg.n_parts();
  // Pose(qbl, tbl).T_.cast<float>(); in the single-LiDAR path the extrinsic of mloam_set_extrinsic, identity without one
  for (int l = 0; l < o->n_lasers; l++) pose_mat12(c->cfg.part_ext(l), o->mat[l]);
}

namespace {

// VoxelGridCovarianceMLOAM<PointI>::filter of a few points, serially (the indexing of pcl::VoxelGrid, voxel_grid_covariance_mloam_impl.hpp
// :84-116, :206-250: bounding box over the finite points, voxel index, a stable sort by index, per voxel the float mean of x, y, z
// accumulated in sorted order and the LAST point's intensity, :417-418,428).  An index space over int32 returns the input (:92-101).
__device__ int voxel_few(const float4 *in, int n, float inv, float4 *out) {
  float mn[3] = {3.4028235e38f, 3.4028235e38f, 3.4028235e38f}, mx[3] = {-3.4028235e38f, -3.4028235e38f, -3.4028235e38f};
  int n_fin = 0;
  for (int i = 0; i < n; i++) {
    const float4 p = in[i];
    if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) continue;
    n_fin++;
    mn[0] = fminf(mn[0], p.x), mn[1] = fminf(mn[1], p.y), mn[2] = fminf(mn[2], p.z);
    mx[0] = fmaxf(mx[0], p.x), mx[1] = fmaxf(mx[1], p.y), mx[2] = fmaxf(mx[2], p.z);
  }
  if (n_fin == 0) return 0;
  const long long dx = (long long)((mx[0] - mn[0]) * inv) + 1, dy = (long long)((mx[1] - mn[1]) * inv) + 1,
                  dz = (long long)((mx[2] - mn[2]) * inv) + 1;
  if (dx * dy * dz > 2147483647ll) {
    for (int i = 0; i < n; i++) out[i] = in[i];
    return n;
  }
  int minb[3], divb[3];
  for (int d = 0; d < 3; d++) {
    minb[d] = (int)floorf(mn[d] * inv);
    divb[d] = (int)floorf(mx[d] * inv) - minb[d] + 1;
  }
  const int mul[3] = {1, divb[0], divb[0] * divb[1]};
  unsigned key[MLOAM_MAX_LIDARS];
  int ord[MLOAM_MAX_LIDARS], m = 0;
  for (int i = 0; i < n; i++) {
    const float4 p = in[i];
    if (!isfinite(p.x) || !isfinite(p.y) || !isfinite(p.z)) continue;
    const int i0 = (int)(floorf(p.x * inv) - (float)minb[0]), i1 = (int)(floorf(p.y * inv) - (float)minb[1]),
              i2 = (int)(floorf(p.z * inv) - (float)minb[2]);
    const unsigned k = (unsigned)(i0 * mul[0] + i1 * mul[1] + i2 * mul[2]);
    int j = m++;  // insertion: equal keys keep their input order
    while (j > 0 && key[j - 1] > k) key[j] = key[j - 1], ord[j] = ord[j - 1], j--;
    key[j] = k, ord[j] = i;
  }
  int n_out = 0;
  for (int a = 0; a < m;) {
    int b = a + 1;
    while (b < m && key[b] == key[a]) b++;
    float sx = 0.f, sy = 0.f, sz = 0.f;
    for (int j = a; j < b; j++) sx = sx + in[ord[j]].x, sy = sy + in[ord[j]].y, sz = sz + in[ord[j]].z;
    const float cnt = (float)(b - a);
    out[n_out++] = make_float4(sx / cnt, sy / cnt, sz / cnt, in[ord[b - 1]].w);
    a = b;
  }
  return n_out;
}

// first[l] / first_ok[l]: the recorded first points; ua (nullable): the frame's with_ua configuration (the gate), else zero cov_vec
__global__ void __launch_bounds__(32) k_outlier_scan(const float4 *__restrict__ first, const int *__restrict__ first_ok, const OutlierStage *__restrict__ cfg,
                                                     const UaStage *__restrict__ ua, float4 *__restrict__ out, float *__restrict__ cov6_out,
                                                     int *__restrict__ n_out) {
  __shared__ float4 raw[MLOAM_MAX_LIDARS], ds[MLOAM_MAX_LIDARS], gated[MLOAM_MAX_LIDARS];
  __shared__ float cov6[6 * MLOAM_MAX_LIDARS], trace[MLOAM_MAX_LIDARS];
  __shared__ int n_ds;
  const int lane = threadIdx.x;
  const int L = cfg->n_lasers;
  if (lane == 0) {
    int n = 0;
    for (int l = 0; l < L; l++) {
      if (!first_ok[l]) continue;  // an empty part pushes no point (laser_cloud_out.points[0] of an empty cloud is not read)
      raw[n++] = rig_transform(cfg->mat[l], first[l], (float)l);  // pcl::transformPointCloud, intensity = n
    }
    n_ds = voxel_few(raw, n, 1.0f / cfg->leaf, ds);
  }
  __syncthreads();
  UctFrame f;
  if (ua) {
    f = ua->frame;
  } else {  // with_ua = false: PointIWithCov(point_ori, Zero) (:407-418)
    memset(&f, 0, sizeof(f));
    f.n_lasers = L, f.scan_frame = 1;
  }
  const int nd = n_ds;
  int keep = 0;
  if (lane < nd) keep = uct_point(ds[lane], f, f.pose_global, ua ? ua->lasers : nullptr, (size_t)lane, gated, cov6, trace);
  const unsigned mask = __ballot_sync(0xffffffffu, keep);
  if (keep) {
    const int o = __popc(mask & ((1u << lane) - 1u));
    out[o] = gated[lane];
#pragma unroll
    for (int k = 0; k < 6; k++) cov6_out[6 * o + k] = cov6[6 * lane + k];
  }
  if (lane == 0) *n_out = __popc(mask);
}

}  // namespace

int outlier_stage(Ctx *c, Ctx::ScanRef *S, const UaStage *d_ua) {
  if (!S->first) return fail(c, MLOAM_E_STATE, "frame: the sweep's first points were not recorded");
  OutlierStage *d_cfg = nullptr;
  float4 *out = nullptr;
  float *cov6 = nullptr;
  int *cnt = nullptr;
  MLOAM_CUDA_OK(c, carve(c->outlier, [&](Carve &cv) {
    d_cfg = cv.take<OutlierStage>(1), out = cv.take<float4>(MLOAM_MAX_LIDARS), cov6 = cv.take<float>(6 * MLOAM_MAX_LIDARS), cnt = cv.take<int>(16);
  }));
  cudaStream_t st = c->stream;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_cfg, &c->pinned->outlier, sizeof(OutlierStage), cudaMemcpyHostToDevice, st));
  k_outlier_scan<<<1, 32, 0, st>>>(S->first, S->first_ok, d_cfg, d_ua, out, cov6, cnt);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  S->outlier = out, S->cov6_outlier = cov6, S->d_n_outlier = cnt;
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

extern "C" {

int mloam_compound_pose_cov(const double *pose1_7, const double *cov1_36, const double *pose2_7, const double *cov2_36, double *pose_out7,
                            double *cov_out36) {
  if (!pose1_7 || !cov1_36 || !pose2_7 || !cov2_36 || !pose_out7 || !cov_out36) return MLOAM_E_INVALID;
  // Pose objects are normalised on construction (pose.cpp:34-41); the product itself is not (associate_uct.hpp:37-38)
  const Q4 q1 = qnormalized(Q4{pose1_7[3], pose1_7[4], pose1_7[5], pose1_7[6]}), q2 = qnormalized(Q4{pose2_7[3], pose2_7[4], pose2_7[5], pose2_7[6]});
  const D3 t1{pose1_7[0], pose1_7[1], pose1_7[2]}, t2{pose2_7[0], pose2_7[1], pose2_7[2]};
  const Q4 q = qmul(q1, q2);
  const D3 t = qrot(q1, t2) + t1;
  pose_out7[0] = t.x, pose_out7[1] = t.y, pose_out7[2] = t.z, pose_out7[3] = q.x, pose_out7[4] = q.y, pose_out7[5] = q.z, pose_out7[6] = q.w;
  H6 c1, c2;
  memcpy(c1.m, cov1_36, sizeof(c1.m)), memcpy(c2.m, cov2_36, sizeof(c2.m));
  const M33 Rm = qmat(q1);
  H3 R, S;
  memcpy(R.m, Rm.m, sizeof(R.m));
  const double sk[9] = {0, -t1.z, t1.y, t1.z, 0, -t1.x, -t1.y, t1.x, 0};
  memcpy(S.m, sk, sizeof(sk));
  H6 Ad;
  memset(Ad.m, 0, sizeof(Ad.m));
  put(Ad, 0, 0, R), put(Ad, 0, 3, h3_mul(S, R)), put(Ad, 3, 3, R);  // adjointMatrix :9-16
  const H6 c2p = h6_mul(h6_mul(Ad, c2), h6_T(Ad));
  const H3 c1rr = blk(c1, 0, 0), c1rp = blk(c1, 0, 3), c1pp = blk(c1, 3, 3), c2rr = blk(c2p, 0, 0), c2rp = blk(c2p, 0, 3), c2pp = blk(c2p, 3, 3);
  H6 A1, A2, B;
  memset(A1.m, 0, sizeof(A1.m)), memset(A2.m, 0, sizeof(A2.m)), memset(B.m, 0, sizeof(B.m));
  put(A1, 0, 0, covop1(c1pp)), put(A1, 0, 3, covop1(h3_add(c1rp, h3_T(c1rp)))), put(A1, 3, 3, covop1(c1pp));
  put(A2, 0, 0, covop1(c2pp)), put(A2, 0, 3, covop1(h3_add(c2rp, h3_T(c2rp)))), put(A2, 3, 3, covop1(c2pp));
  const H3 Brr = h3_add(h3_add(h3_add(covop2(c1pp, c2rr), covop2(h3_T(c1rp), c2rp)), covop2(c1rp, h3_T(c2rp))), covop2(c1rr, c2pp));
  const H3 Brp = h3_add(covop2(c1pp, h3_T(c2rp)), covop2(h3_T(c1rp), c2pp));
  put(B, 0, 0, Brr), put(B, 0, 3, Brp), put(B, 3, 0, h3_T(Brp)), put(B, 3, 3, covop2(c1pp, c2pp));
  const H6 u1 = h6_mul(A1, c2p), u2 = h6_mul(c2p, h6_T(A1)), u3 = h6_mul(A2, c1), u4 = h6_mul(c1, h6_T(A2));
  for (int i = 0; i < 36; i++) cov_out36[i] = c1.m[i] + c2p.m[i] + (((u1.m[i] + u2.m[i]) + u3.m[i]) + u4.m[i]) / 12 + B.m[i] / 4;
  return MLOAM_OK;
}

int mloam_cloud_uct_associate(mloam_ctx_t *h, const mloam_point_t *h_pts, int n, const double *pose_global7, int n_lasers, const double *ext7,
                              const double *pose_compound7, const double *cov_compound36, const double *cov_meas9, int with_ua,
                              double trace_threshold, mloam_point_t *h_out, float *h_cov6_out, float *h_trace_out, int *n_out) {
  if (!h || n < 0 || !pose_global7 || n_lasers < 1 || n_lasers > MLOAM_MAX_LIDARS || !ext7 || !pose_compound7 || !cov_compound36 || !cov_meas9 ||
      !n_out || (n > 0 && (!h_pts || !h_out || !h_cov6_out || !h_trace_out)))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_out = 0;
  if (n == 0) return MLOAM_OK;
  cudaStream_t st = c->stream;
  UctBufs B;
  int rc = uct_bufs(c, n, &B);
  if (rc) return rc;
  const size_t N1 = (size_t)n + 16;
  float4 *d_in, *d_out;
  UctLaser *d_l;
  float *d_c6, *d_tr;
  int *d_total;
  MLOAM_CUDA_OK(c, carve(c->sweep_in, [&](Carve &cv) { d_in = cv.take<float4>(n), d_l = cv.take<UctLaser>(MLOAM_MAX_LIDARS); }));
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) {
    d_out = cv.take<float4>(N1), d_c6 = cv.take<float>(6 * N1), d_tr = cv.take<float>(N1), d_total = cv.take<int>(16);
  }));
  std::vector<UctLaser> L;
  fill_lasers(n_lasers, ext7, pose_compound7, cov_compound36, L);
  UctFrame f;
  memcpy(f.pose_global, pose_global7, sizeof(f.pose_global)), memcpy(f.cov_meas, cov_meas9, sizeof(f.cov_meas));
  f.trace_threshold = trace_threshold, f.with_ua = with_ua ? 1 : 0, f.n_lasers = n_lasers, f.scan_frame = 0;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_in, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_l, L.data(), sizeof(UctLaser) * n_lasers, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(d_total, 0, sizeof(int), st));
  rc = uct_associate_append(c, d_in, n, f, d_l, B, d_out, d_c6, d_tr, d_total);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_total, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));  // L (host vector) was read by the copy above
  *n_out = hc[0];
  if (hc[0] > 0) {
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6_out, d_c6, sizeof(float) * 6 * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_trace_out, d_tr, sizeof(float) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  }
  return MLOAM_OK;
}

int mloam_voxel_downsample_cov(mloam_ctx_t *h, const mloam_point_t *h_pts, const float *h_cov6, const float *h_trace, int n, float leaf,
                               float trace_threshold, mloam_point_t *h_out, float *h_cov6_out, float *h_trace_out, int *n_out) {
  if (!h || n < 0 || !n_out || !(leaf > 0.f) || (n > 0 && (!h_pts || !h_cov6 || !h_trace || !h_out || !h_cov6_out || !h_trace_out))) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  *n_out = 0;
  if (n == 0) return MLOAM_OK;
  cudaStream_t st = c->stream;
  const size_t N1 = (size_t)n + 16;
  float4 *d_in, *d_out;
  float *d_c6, *d_tr, *d_oc6, *d_otr;
  int *d_cnt;
  MLOAM_CUDA_OK(c, carve(c->sweep_in, [&](Carve &cv) { d_in = cv.take<float4>(N1), d_c6 = cv.take<float>(6 * N1), d_tr = cv.take<float>(N1); }));
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) {
    d_out = cv.take<float4>(N1), d_oc6 = cv.take<float>(6 * N1), d_otr = cv.take<float>(N1), d_cnt = cv.take<int>(16);
  }));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_in, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_c6, h_cov6, sizeof(float) * 6 * (size_t)n, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_tr, h_trace, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, st));
  int rc = voxel_downsample_cov_device(c, d_in, d_c6, d_tr, n, nullptr, leaf, trace_threshold, d_out, d_oc6, d_otr, d_cnt, c->voxel_work);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  *n_out = hc[0];
  if (hc[0] > 0) {
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6_out, d_oc6, sizeof(float) * 6 * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_trace_out, d_otr, sizeof(float) * (size_t)hc[0], cudaMemcpyDeviceToHost, st));
    MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  }
  return MLOAM_OK;
}

int mloam_submap_assemble(mloam_ctx_t *h, int slot, int n_keyframes, const mloam_point_t *h_pts, const int *counts, const double *poses7, int n_lasers,
                          const double *ext7, const double *pose_compound7, const double *cov_compound36, const double *cov_meas9, int with_ua,
                          double trace_threshold_assoc, float leaf, float trace_threshold_filter, float map_cell, mloam_point_t *h_out,
                          float *h_cov6_out, int *n_out) {
  if (!h || slot < 0 || slot >= MLOAM_NUM_MAPS || n_keyframes < 0 || !counts || !poses7 || n_lasers < 1 || n_lasers > MLOAM_MAX_LIDARS || !ext7 ||
      !pose_compound7 || !cov_compound36 || !cov_meas9 || !(leaf > 0.f))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (n_out) *n_out = 0;
  size_t n_total = 0;
  int n_max = 0;
  for (int k = 0; k < n_keyframes; k++) {
    if (counts[k] < 0) return MLOAM_E_INVALID;
    n_total += (size_t)counts[k], n_max = counts[k] > n_max ? counts[k] : n_max;
  }
  if (n_total > 0 && !h_pts) return MLOAM_E_INVALID;
  if (n_total > 0x7fffff00ull) return fail(c, MLOAM_E_INVALID, "submap_assemble: more than 2^31 points");
  const int n = (int)n_total;
  cudaStream_t st = c->stream;
  UctBufs B;
  int rc = uct_bufs(c, n_max, &B);
  if (rc) return rc;
  const size_t N1 = (size_t)n + 16;
  float4 *d_in, *d_mid, *d_fin;
  UctLaser *d_l;
  float *d_mc6, *d_mtr, *d_fc6, *d_ftr;
  int *d_total, *d_cnt;
  MLOAM_CUDA_OK(c, carve(c->sweep_in, [&](Carve &cv) {
    d_in = cv.take<float4>(N1), d_l = cv.take<UctLaser>(MLOAM_MAX_LIDARS * (size_t)(n_keyframes + 1));
  }));
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) {
    d_mid = cv.take<float4>(N1), d_mc6 = cv.take<float>(6 * N1), d_mtr = cv.take<float>(N1), d_total = cv.take<int>(16);
  }));
  MLOAM_CUDA_OK(c, carve(c->host_work, [&](Carve &cv) {
    d_fin = cv.take<float4>(N1), d_fc6 = cv.take<float>(6 * N1), d_ftr = cv.take<float>(N1), d_cnt = cv.take<int>(16);
  }));
  // all keyframe clouds and all per-(keyframe, LiDAR) compound poses go up in two copies
  std::vector<UctLaser> L((size_t)n_keyframes * n_lasers);
  for (int k = 0; k < n_keyframes; k++) {
    std::vector<UctLaser> one;
    fill_lasers(n_lasers, ext7, pose_compound7 + 7 * (size_t)k * n_lasers, cov_compound36 + 36 * (size_t)k * n_lasers, one);
    for (int l = 0; l < n_lasers; l++) L[(size_t)k * n_lasers + l] = one[l];
  }
  if (n > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_in, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  if (!L.empty()) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_l, L.data(), sizeof(UctLaser) * L.size(), cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemsetAsync(d_total, 0, sizeof(int), st));
  size_t off = 0;
  for (int k = 0; k < n_keyframes; k++) {  // `+=` keyframe after keyframe (:338-342)
    UctFrame f;
    memcpy(f.pose_global, poses7 + 7 * (size_t)k, sizeof(f.pose_global)), memcpy(f.cov_meas, cov_meas9, sizeof(f.cov_meas));
    f.trace_threshold = trace_threshold_assoc, f.with_ua = with_ua ? 1 : 0, f.n_lasers = n_lasers, f.scan_frame = 0;
    rc = uct_associate_append(c, d_in + off, counts[k], f, d_l + (size_t)k * n_lasers, B, d_mid, d_mc6, d_mtr, d_total);
    if (rc) return rc;
    off += (size_t)counts[k];
  }
  // VoxelGridCovarianceMLOAM over the merged cloud (:344-347): the merged size is only known on the device
  rc = voxel_downsample_cov_device(c, d_mid, d_mc6, d_mtr, n, d_total, leaf, trace_threshold_filter, d_fin, d_fc6, d_ftr, d_cnt, c->voxel_work);
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));  // the map build is sized by the submap's point count
  const int m = hc[0];
  if (n_out) *n_out = m;
  rc = map_build_device(c, slot, d_fin, m, pick_cell(c, map_cell));  // kdtree->setInputCloud on the assembled submap, device to device
  if (rc) return rc;
  if (m > 0 && h_out) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_fin, sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, st));
  if (m > 0 && h_cov6_out) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_cov6_out, d_fc6, sizeof(float) * 6 * (size_t)m, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

// Estimator::buildLocalMap / buildCalibMap, the map half (estimator.cpp:1175-1204 / :1084-1110) for one LiDAR and one feature kind: the
// window's stacked clouds (sensor frame) -> pivot frame with pose_local[i] -> `+=` -> pcl::VoxelGrid(leaf) -> map slot.
int mloam_local_map_build(mloam_ctx_t *h, int slot, int n_frames, const mloam_point_t *h_pts, const int *counts, const double *pose_local7, float leaf,
                          float map_cell, mloam_point_t *h_out, int *n_out) {
  if (!h || slot < 0 || slot >= MLOAM_NUM_MAPS || n_frames < 0 || n_frames > 64 || !counts || !pose_local7 || !(leaf > 0.f)) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (n_out) *n_out = 0;
  std::vector<int> off(n_frames + 1, 0);
  for (int k = 0; k < n_frames; k++) {
    if (counts[k] < 0) return MLOAM_E_INVALID;
    off[k + 1] = off[k] + counts[k];
  }
  const int n = off[n_frames];
  if (n > 0 && !h_pts) return MLOAM_E_INVALID;
  cudaStream_t st = c->stream;
  std::vector<float> mats(12 * (size_t)(n_frames + 1), 0.f);
  for (int k = 0; k < n_frames; k++) pose_mat12(pose_local7 + 7 * (size_t)k, &mats[12 * (size_t)k]);  // Pose(Matrix4d) normalises q
  const size_t N1 = (size_t)n + 16;
  float4 *d_in, *d_out;
  int *d_off, *d_cnt;
  float *d_mat;
  MLOAM_CUDA_OK(c, carve(c->sweep_in, [&](Carve &cv) { d_in = cv.take<float4>(N1), d_off = cv.take<int>(off.size()), d_mat = cv.take<float>(mats.size()); }));
  MLOAM_CUDA_OK(c, carve(c->map_in[0], [&](Carve &cv) { d_out = cv.take<float4>(N1), d_cnt = cv.take<int>(16); }));
  if (n > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_in, h_pts, sizeof(float4) * (size_t)n, cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_off, off.data(), sizeof(int) * off.size(), cudaMemcpyHostToDevice, st));
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_mat, mats.data(), sizeof(float) * mats.size(), cudaMemcpyHostToDevice, st));
  int rc = transform_segments_device(c, d_in, n, d_off, n_frames, d_mat);
  if (rc) return rc;
  rc = voxel_downsample_device(c, d_in, n, nullptr, leaf, 0, d_out, d_cnt, c->voxel_work);  // pcl::VoxelGrid<PointI>: every field averaged
  if (rc) return rc;
  int *hc = c->pinned->counts;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hc, d_cnt, sizeof(int), cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));  // also: the host vectors above have been consumed
  const int m = hc[0];
  if (n_out) *n_out = m;
  rc = map_build_device(c, slot, d_out, m, pick_cell(c, map_cell));
  if (rc) return rc;
  if (m > 0 && h_out) MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_out, d_out, sizeof(float4) * (size_t)m, cudaMemcpyDeviceToHost, st));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(st));
  return MLOAM_OK;
}

}  // extern "C"
