// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The mapper-side frame of lidar_mapper_keyframe.cpp with its options, as flat C entry points of liborc.so:
//   with_ua (orc_frame_ua with ext_cov36): downsampleCurrentScan's uncertainty gate (:356-421, orc_capi.hpp's ua_gate);
//     sqrt_info of every residual from its point's covariance (extractCov + clamp, :541-560, lidar_map_factor.hpp:34,41);
//     cov_mapping = mat_H.inverse() after the last Solve (:600-610): H = problem.Evaluate at the returned pose with the residual blocks
//     of the last association;
//   the DISTORTION step of the odometry (orc_frame_ua with poses7; orc_capi.cpp's orc_undist_points, orc_undist_poses):
//     Estimator::process estimator.cpp:575-579: pose_undist[n] = Pose(qbl_n, tbl_n).inverse() * pose_rlt_[IDX_REF] * Pose(qbl_n, tbl_n)
//     (Pose::inverse / operator*, pose.cpp:99-113, every Pose normalising its quaternion); undistortMeasurements :376-408 with
//     TransformToEnd (orc_capi.hpp) on corner_points_less_sharp and surf_points_less_flat, pose_undist[n] when ESTIMATE_EXTRINSIC == 2,
//     else pose_undist[IDX_REF]; sharp, flat and the outlier cloud untouched.  Without the rig merge (ext7 == nullptr): the whole
//     sweep's extractCloud, the step, and pointAssociateToMap with the single extrinsic (mloam_set_extrinsic);
//   the outlier cloud of segment_cloud: 0 (orc_outlier_frame, laser_cloud_outlier_cov): ImageSegmenter::segmentCloud
//     image_segmenter.hpp:390 gives ONE point per LiDAR, laser_cloud_out.points[0], the first point of its ring-ordered cloud (none for
//     an empty cloud, mloam_adapter.hpp:114 skips the undefined read); pubPointCloud's float transform with intensity = n
//     (visualization.cpp:40-52, :89-104); downsampleCurrentScan :366-368, :407-418: VoxelGridCovarianceMLOAM<PointI>(MAP_OUTLIER_RES)
//     (:1283-1284), then with with_ua the scans' gate, cov_vec zero without it.
// Restatement choices (in addition to orc_math.hpp's):
//   - the 6x6 inverse is an unblocked partial-pivot LU (first largest |pivot| of the column, row swap, multipliers divided by the
//     pivot, rank-1 update of the trailing block) solved column by column — Eigen's algorithm, not its blocked kernels;
//   - when the last evaluation has no residual rows the covariance is zero, where Eigen would return inf / NaN;
//   - the last association is recovered by re-running orc::scan2map with one GN iteration fewer (deterministic) and matching at its
//     pose, so the restatement of the Solve itself stays the one of orc_pipeline.hpp;
//   - LiDAR l's part of a frame's concatenation is [scan_start[l R] - 5, scan_start[(l + 1) R] - 5) (the last one ends at n), as
//     prepare_multi cuts it.
#include "orc_capi.hpp"

using namespace orc;

extern "C" {

// ---- the mapper-side frame (orc_capi.hpp's frame_ua): with_ua when ext_cov36 is set, the undistortion when poses7 is set, the
// single-LiDAR path when ext7 is nullptr.
void orc_frame_ua(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                  const double *single_ext7, const double *poses7, float scan_period, const double *ext_cov36, const double *cov_meas9,
                  double trace_threshold, const float *surf_map, int n_sm, const float *corner_map, int n_cm, float corner_leaf,
                  float surf_leaf, const double *pose_init7, const double *opts, double *pose_out7, double *stats, double *cov36,
                  double *H36, float *surf_out, float *surf_cov6, int *n_surf, float *corner_out, float *corner_cov6, int *n_corner) {
  frame_ua(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, single_ext7, poses7, scan_period, ext_cov36, cov_meas9, trace_threshold,
           surf_map, n_sm, corner_map, n_cm, corner_leaf, surf_leaf, pose_init7, opts, pose_out7, stats, cov36, H36, surf_out, surf_cov6, n_surf,
           corner_out, corner_cov6, n_corner);
}

// ---- the rig frame with with_ua = true: orc_frame_ua without the undistortion.  ext_cov36: n_lidars x 36.
void orc_ua_frame_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                        const double *ext_cov36, const double *cov_meas9, double trace_threshold, const float *surf_map, int n_sm,
                        const float *corner_map, int n_cm, float corner_leaf, float surf_leaf, const double *pose_init7, const double *opts,
                        double *pose_out7, double *stats, double *cov36, double *H36, float *surf_out, float *surf_cov6, int *n_surf,
                        float *corner_out, float *corner_cov6, int *n_corner) {
  frame_ua(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, nullptr, nullptr, 0.f, ext_cov36, cov_meas9, trace_threshold, surf_map, n_sm,
           corner_map, n_cm, corner_leaf, surf_leaf, pose_init7, opts, pose_out7, stats, cov36, H36, surf_out, surf_cov6, n_surf, corner_out,
           corner_cov6, n_corner);
}

// laser_cloud_outlier_cov of a rig frame (the inputs of orc_frame_ua): out (capacity n_lidars points) and cov6, *n_out.
// ext_cov36 (n_lidars x 36) is read with with_ua only.
void orc_outlier_frame(const float *cloud, int n, const int *scan_start, int n_scans, int n_lidars, const double *ext7, const double *ext_cov36,
                       const double *cov_meas9, int with_ua, double trace_threshold, float leaf, float *out, float *out_cov6, int *n_out) {
  const int R = n_scans / n_lidars;
  Cloud raw;
  for (int l = 0; l < n_lidars; l++) {
    const int lo = scan_start[l * R] - 5, hi = (l + 1 < n_lidars) ? scan_start[(l + 1) * R] - 5 : n;
    if (!(lo < hi) || lo < 0 || lo >= n) continue;  // an empty part pushes no point
    raw.push_back(FloatTransform(ext7 + 7 * l)(to_cloud(cloud + 4 * (size_t)lo, 1)[0], (float)l));
  }
  Cloud ds, o;
  voxel_grid(raw, leaf, ds, true);
  std::vector<float> c6;
  ua_gate(ds, ext7, with_ua ? ext_cov36 : nullptr, cov_meas9, trace_threshold, o, c6, nullptr);
  *n_out = (int)o.size();
  if (!o.empty()) std::memcpy(out, o.data(), sizeof(PointI) * o.size()), std::memcpy(out_cov6, c6.data(), sizeof(float) * c6.size());
}

// ---- scan2MapOptimization with per-point cov_vec (as orc_scan2map_ua) that also reports cov_mapping and the H it inverts
void orc_ua_scan2map(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_scan, int n_ss, const float *surf_cov6,
                     const float *corner_scan, int n_cs, const float *corner_cov6, const double *pose_init7, const double *opts, double *pose_out7,
                     double *stats, double *cov36, double *H36) {
  Scan2MapOptions o = opts_from(opts);
  std::vector<double> ts(n_ss), tc(n_cs);
  for (int i = 0; i < n_ss; i++) ts[i] = (double)surf_cov6[i * 6] + (double)surf_cov6[i * 6 + 3] + (double)surf_cov6[i * 6 + 5];
  for (int i = 0; i < n_cs; i++) tc[i] = (double)corner_cov6[i * 6] + (double)corner_cov6[i * 6 + 3] + (double)corner_cov6[i * 6 + 5];
  o.surf_cov_trace = &ts, o.corner_cov_trace = &tc;
  double cov[36], H[36];
  Scan2MapResult r = scan2map_with_cov(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), to_cloud(surf_scan, n_ss), to_cloud(corner_scan, n_cs),
                                       to_pose(pose_init7), o, cov, H);
  pose_to_param(r.pose, pose_out7);
  if (stats) stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
  if (cov36) std::memcpy(cov36, cov, sizeof(cov));
  if (H36) std::memcpy(H36, H, sizeof(H));
}

}  // extern "C"
