/* mloam_b200.h — C ABI of the H100-native M-LOAM per-scan hot path.
 *
 * Plain C, POD only, no torch / Eigen / PCL / Ceres types.  Every entry point names the reference
 * interface (file:line, relative to gogojjh/M-LOAM) it replaces.  All functions return 0 on success
 * and a negative MLOAM_E_* code otherwise; mloam_last_error() gives the text.  There is no CPU
 * fallback: with no CUDA device mloam_ctx_create() fails with MLOAM_E_NO_DEVICE.
 *
 * One context == one CUDA device + one stream + grow-only device arenas.  A context is not shared
 * between host threads (the reference calls extractCloud/trackCloud from one OpenMP thread per LiDAR,
 * estimator.cpp:249,423 — use one context per thread).
 *
 * Pointers named h_* are HOST buffers (pinned optional); d_* are DEVICE buffers on the context's
 * device.  Points are float4 (x, y, z, intensity) == the payload of pcl::PointXYZI
 * (common::PointI, mloam_common/libs/include/common/types/type.h:20); intensity = ring id + relative
 * time (image_segmenter.hpp:128).  Poses are 7 doubles [tx ty tz qx qy qz qw]
 * (pose_local_parameterization.h:20).
 */
#ifndef MLOAM_B200_H_
#define MLOAM_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MLOAM_OK 0
#define MLOAM_E_INVALID (-1)   /* bad argument */
#define MLOAM_E_NO_DEVICE (-2) /* no CUDA device / wrong architecture */
#define MLOAM_E_CUDA (-3)      /* CUDA runtime error, see mloam_last_error */
#define MLOAM_E_STATE (-4)     /* call order (e.g. match before map build) */
#define MLOAM_E_NCCL (-5)

#define MLOAM_MAP_CORNER 0 /* kdtree_corner_from_map, lidar_mapper_keyframe.cpp:434 */
#define MLOAM_MAP_SURF 1   /* kdtree_surf_from_map,   lidar_mapper_keyframe.cpp:433 */
#define MLOAM_NUM_MAPS 4   /* 2,3: scan-to-scan targets (lidar_tracker.cpp:33-34) */
#define MLOAM_MAP_SCAN_CORNER 2
#define MLOAM_MAP_SCAN_SURF 3

typedef struct mloam_ctx mloam_ctx_t;

typedef struct {
  float x, y, z, intensity;
} mloam_point_t;

/* The globals of estimator/src/estimator/parameters.h:45-133 that steer the path, plus the hard-coded
 * constants of the orchestrators, as one POD (defaults: mloam_default_params). */
typedef struct {
  int n_scans;                 /* N_SCANS */
  float distance_sq_threshold; /* DISTANCE_SQ_THRESHOLD, feature_extract.hpp:158 */
  float nearby_scan;           /* NEARBY_SCAN,           feature_extract.hpp:171 */
  float min_match_sq_dis;      /* MIN_MATCH_SQ_DIS,      feature_extract.hpp:667 */
  float min_plane_dis;         /* MIN_PLANE_DIS,         feature_extract.hpp:832 */
  int n_neigh;                 /* N_NEIGH (5; lidar_mapper.h:253) */
  int check_fov;               /* CHECK_FOV (false for all *PointFromMap callers) */
  int point_plane_factor;      /* POINT_PLANE_FACTOR */
  int point_edge_factor;       /* POINT_EDGE_FACTOR */
  double huber_a;              /* ceres::HuberLoss(0.1), lidar_mapper_keyframe.cpp:443 */
  double eig_thre;             /* MAP_EIG_THRE, lidar_mapper_keyframe.cpp:1180 */
  double cov_trace;            /* trace(COV_MEASUREMENT) when with_ua=false, :541-545 */
  int max_outer;               /* max_iter = 2, lidar_mapper_keyframe.cpp:439 */
  int max_inner;               /* options.max_num_iterations = 30, :590 */
  float map_cell;              /* voxel-hash cell edge [m] for the scan-to-map maps (<= 0: auto) */
  float corner_leaf;           /* MAP_CORNER_RES (scan down-sampling before matching) */
  float surf_leaf;             /* MAP_SURF_RES */
  int gf_method;               /* FLAGS_gf_method in scan2MapOptimization (:474-532): 0 wo_gf, 1 rnd, 2 fps, 3 gd_fix */
  float gf_ratio;              /* FLAGS_gf_ratio_ini */
  unsigned gf_seed;            /* selection seed; outer iteration i, set s (0 corner, 1 surf) uses gf_seed + 2 i + s */
  int max_ring_points;         /* upper bound of the points of one ring (0: up to 12288); sizes the in-CTA sort of extractCloud so that
                                  several rings share an SM — set it to the sensor's horizontal resolution */
  int reserved[4];
} mloam_params_t;

/* Per-solve report (what the reference prints through summary.BriefReport / timers). */
typedef struct {
  int ran;            /* 0 when the map-size gate (lidar_mapper_keyframe.cpp:429) rejected the frame */
  int n_surf;         /* matched surf features, last outer iteration */
  int n_corner;       /* matched corner features, last outer iteration */
  int lm_iterations;  /* LM iterations over all outer iterations */
  int degenerate;     /* PoseLocalParameterization::is_degenerate_ of the last outer iteration */
  int termination;    /* last Solve: 0 max-iter, 1 function tol, 2 parameter tol, 3 gradient tol, 4 failure, 5 too few correspondences (iteration skipped),
                       * 8 the two-evaluation launch timed out at its grid barrier (MLOAM_E_STATE), 9 peer-memory exchange failed (MLOAM_E_NCCL) */
  double final_cost;
  double eig[6];      /* eigenvalues of J^T J (evalDegenracy) of the last outer iteration */
  double H[36];       /* loss-corrected J^T J evaluated before the last Solve (:575-581) */
  int n_surf_in;      /* features that entered matching (after scan down-sampling) */
  int n_corner_in;
  int reserved[6];
} mloam_solve_stats_t;

/* Feature sets of FeatureExtract::extractCloud (cloudFeature, parameters.h:161). Host buffers are
 * caller-owned with capacity cap points each (cap >= n input points is always enough). */
typedef struct {
  mloam_point_t *corner_points_sharp;
  mloam_point_t *corner_points_less_sharp;
  mloam_point_t *surf_points_flat;
  mloam_point_t *surf_points_less_flat;
  int n_sharp, n_less_sharp, n_flat, n_less_flat;
  int cap;
} mloam_features_t;

/* ---- context -------------------------------------------------------------------------------- */
void mloam_default_params(mloam_params_t *p);
int mloam_ctx_create(int device, const mloam_params_t *params, mloam_ctx_t **out);
void mloam_ctx_destroy(mloam_ctx_t *ctx);
int mloam_set_params(mloam_ctx_t *ctx, const mloam_params_t *params);
/* Run on an external CUDA stream (cudaStream_t passed as void*), e.g. torch's current stream. */
int mloam_set_stream(mloam_ctx_t *ctx, void *cuda_stream);
int mloam_sync(mloam_ctx_t *ctx);
const char *mloam_last_error(mloam_ctx_t *ctx);
const char *mloam_version(void);
/* Kernels launched by this context since creation (bench's gpu_launches). */
long long mloam_launch_count(mloam_ctx_t *ctx);
/* Per-kernel device timing with CUDA events on the context stream.  name: "map_build", "match",
 * "linearize", "lm", "extract", "voxel".  Returns total ms and launch count since the last reset. */
int mloam_profile_enable(mloam_ctx_t *ctx, int on);
int mloam_profile_get(mloam_ctx_t *ctx, const char *name, double *ms_total, long long *launches);
int mloam_profile_reset(mloam_ctx_t *ctx);

/* ---- ImageSegmenter::segmentCloud with ScanInfo::segment_flag_ == false (`segment_cloud: 0`): the range-image projection
 *      (image_segmenter.hpp:88-136) and the ring-ordered output + ScanInfo (:381-389) that feed extractCloud (estimator.cpp:122,228,258).
 *      vertical_scans 16 / 32 / 64 and horizon_scans as ImageSegmenter::setParameter takes them (image_segmenter.cpp:18-63); roi_range = ROI_RANGE
 *      (parameters.cpp:211).  h_out holds up to n points (intensity += ring id), h_scan_start / h_scan_end hold vertical_scans entries each.
 *      The BFS labelling of segment_cloud: 1 (image_segmenter.hpp:160-360) is not provided. */
int mloam_project_cloud(mloam_ctx_t *ctx, const mloam_point_t *h_cloud, int n, int vertical_scans, int horizon_scans, double roi_range,
                        mloam_point_t *h_out, int *n_out, int *h_scan_start, int *h_scan_end);

/* ---- raw driver sweeps: the three steps before extractCloud in Estimator::inputCloud (estimator.cpp:249-261), per LiDAR —
 *      pcl::removeNaNFromPointCloud in the driver node (rosNodeRVKITTI.cpp:154-161, rosNodeRVOxford.cpp:170-177), then
 *      FeatureExtract::calTimestamp (feature_extract.cpp:25-114), then segmentCloud with segment_cloud: 0 (as mloam_project_cloud).
 * mloam_cal_timestamp: removeNaN + calTimestamp of ONE LiDAR's sweep: h_out (capacity n) receives the points with a finite x, y and z, in
 *   input order, intensity = relative time; *n_out their count.  time_field 0: the time from the azimuth (calTimestamp(PointCloud),
 *   :54-114: -atan2 of the first and last point, the half_passed wrap, (ori - start) / (end - start) * scan_period); time_field 1: from the
 *   point's timestamp field in microseconds carried in the intensity lane (calTimestamp(PointITimeCloud), :38-52: timestamp * 1e-6).  The
 *   cloud's own intensity is discarded either way.  scan_period = SCAN_PERIOD (parameters.h:78).
 * mloam_set_front_end: the front end of mloam_frame_raw*: vertical_scans 16 / 32 / 64, horizon_scans and roi_range as mloam_project_cloud
 *   takes them, scan_period and time_field as mloam_cal_timestamp.  MLOAM_E_INVALID for another vertical_scans, and when a nonzero
 *   params.max_ring_points is below horizon_scans (a projected ring holds up to horizon_scans points).
 * mloam_frame_raw / mloam_frame_raw_device: mloam_frame / mloam_frame_device on the rig's RAW sweeps, concatenated LiDAR-major, h_counts[l]
 *   points of LiDAR l (n_lidars of mloam_set_lidars, one without it; counts always in host memory).  Per LiDAR removeNaN + calTimestamp +
 *   projection onto a range image of its own run on the device, batched over the rig; the ring-ordered sweep (LiDAR-major, ring-major,
 *   n_lidars x vertical_scans rings of ScanInfo) goes to extractCloud without a host round trip.  Results are identical to mloam_frame* on
 *   the concatenation of the per-LiDAR mloam_cal_timestamp + mloam_project_cloud outputs with the ScanInfo offset by each LiDAR's start.
 *   with_ua, the keyframe store, mloam_frame_scan and mloam_pose_covariance work as after mloam_frame.  MLOAM_E_INVALID when a count is 0
 *   (the node's empty_check, rosNodeRVOxford.cpp:216-220); MLOAM_E_STATE without mloam_set_front_end and on a context with a communicator.
 *   The check is on the counts as passed: a LiDAR whose points are ALL non-finite passes it and contributes empty rings to the frame,
 *   whereas the node runs removeNaNFromPointCloud before empty_check (rosNodeRVOxford.cpp:175, :216-220) and skips that frame.  Counting
 *   the finite points would need a device-to-host read-back before the frame; a caller that can receive such sweeps checks them itself
 *   (mloam_cal_timestamp returns the finite count). 
 * mloam_front_end: the front end of mloam_frame_raw alone, host-in / host-out: h_out (capacity = sum of counts) receives the ring-ordered
 *   sweep, *n_out its size, h_scan_start / h_scan_end the n_lidars x vertical_scans rings of its ScanInfo.
 * mloam_frame_set_next_raw / mloam_frame_set_next_raw_device: the look-ahead of mloam_frame_set_next* for raw sweeps (the front end runs in
 *   the look-ahead branch too); picked up by the next mloam_frame_raw* call with the same pointer and counts.  NULL withdraws. */
int mloam_cal_timestamp(mloam_ctx_t *ctx, const mloam_point_t *h_cloud, int n, int time_field, float scan_period, mloam_point_t *h_out,
                        int *n_out);
int mloam_set_front_end(mloam_ctx_t *ctx, int vertical_scans, int horizon_scans, double roi_range, float scan_period, int time_field);
int mloam_front_end(mloam_ctx_t *ctx, const mloam_point_t *h_raw, const int *h_counts, mloam_point_t *h_out, int *n_out, int *h_scan_start,
                    int *h_scan_end);
int mloam_frame_raw(mloam_ctx_t *ctx, const mloam_point_t *h_raw, const int *h_counts, const mloam_point_t *h_surf_map, int n_surf_map,
                    const mloam_point_t *h_corner_map, int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                    mloam_solve_stats_t *stats);
int mloam_frame_raw_device(mloam_ctx_t *ctx, const mloam_point_t *d_raw, const int *h_counts, const mloam_point_t *d_surf_map,
                           int n_surf_map, const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps,
                           const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats);
int mloam_frame_set_next_raw(mloam_ctx_t *ctx, const mloam_point_t *h_raw, const int *h_counts);
int mloam_frame_set_next_raw_device(mloam_ctx_t *ctx, const mloam_point_t *d_raw, const int *h_counts);

/* ---- FeatureExtract::extractCloud (feature_extract.cpp:118-297) -------------------------------- */
int mloam_extract_features(mloam_ctx_t *ctx, const mloam_point_t *h_cloud, int n, const int *h_scan_start,
                           const int *h_scan_end, int n_scans, mloam_features_t *out);
/* Optional per-point by-products of the last extraction (curvature feature_extract.cpp:138, label :141). */
int mloam_extract_debug(mloam_ctx_t *ctx, float *h_curvature, int *h_label, int n);

/* ---- pcl::VoxelGrid<PointI>::filter (feature_extract.cpp:267-270, estimator.cpp:488-494) and
 *      VoxelGridCovarianceMLOAM on plain points (intensity_last=1; lidar_mapper_keyframe.cpp:359-368) */
int mloam_voxel_downsample(mloam_ctx_t *ctx, const mloam_point_t *h_in, int n, float leaf, int intensity_last,
                           mloam_point_t *h_out, int *n_out);

/* ---- pcl::KdTreeFLANN::setInputCloud (lidar_mapper_keyframe.cpp:433-434, lidar_tracker.cpp:33-34,
 *      estimator.cpp:1129-1130,1231-1233): build the GPU voxel-hash over a cloud. */
int mloam_map_build(mloam_ctx_t *ctx, int slot, const mloam_point_t *h_pts, int m, float cell);
int mloam_map_build_device(mloam_ctx_t *ctx, int slot, const mloam_point_t *d_pts, int m, float cell);
int mloam_map_size(mloam_ctx_t *ctx, int slot);

/* ---- pcl::KdTreeFLANN::nearestKSearch (feature_extract.hpp:155,293,406,570,666,813): exact K nearest
 * within sqrt(max_sqdist), ascending (squared distance, index).  Queries are transformed by pose7 first
 * when it is non-null (pointAssociateToMap, utility.h:103-117).  Slots with no neighbour inside the
 * radius get idx -1 / sqdist +inf.  k in {1,5,10}. */
int mloam_knn(mloam_ctx_t *ctx, int slot, const mloam_point_t *h_q, int nq, const double *pose7, int k,
              float max_sqdist, int *h_idx, float *h_sqdist);

/* ---- FeatureExtract::matchCornerFromMap / matchSurfFromMap (feature_extract.hpp:378-643; per-point
 * forms :645-883).  type 'c' | 's'.  Outputs per query i: valid[i]; coeffs[i*6..] ('c': [X1;X2], 's':
 * (n,d,0,0)); nn[i*n_neigh..] neighbour indices (may be null). */
int mloam_match_from_map(mloam_ctx_t *ctx, int slot, int type, const mloam_point_t *h_pts, int n, const double *pose7,
                         unsigned char *h_valid, double *h_coeffs, int *h_nn);

/* ---- Lidar*Factor::Evaluate, batched (lidar_map_factor.hpp:44-68,143-171; lidar_scan_factor.hpp:33-60,
 * 245-279; lidar_pure_odom_factor.hpp:38-101,209-281; lidar_online_calib_factor.hpp:34-60,135-163).
 * kind: 0 plane (1x7), 1 edge scalar (1x7), 2 edge 3-vector (3x7), 3 odom plane (1x21 = [pivot|i|ext]),
 * 4 odom edge (1x21).  points n*3, coeffs n*6, sqrt_info n (null = 1).  params: 7 doubles (kinds 0-2) or
 * 21 (kinds 3-4), shared by the batch.  residuals n*rows; jacobians n*rows*cols row-major (may be null). */
int mloam_factor_evaluate(mloam_ctx_t *ctx, int kind, int n, const double *h_points, const double *h_coeffs,
                          const double *h_sqrt_info, const double *h_params, double *h_residuals,
                          double *h_jacobians);

/* ---- normal equations of a single-pose problem (what Ceres assembles inside Solve / what
 * problem.Evaluate -> evalHessian returns, lidar_mapper_keyframe.cpp:575-581,1160-1169): types[n] 's'|'c',
 * Huber-corrected J^T J (6x6 row-major), J^T r, cost = 1/2 sum rho. */
int mloam_normal_equations(mloam_ctx_t *ctx, int n, const unsigned char *h_types, const double *h_points,
                           const double *h_coeffs, double sqrt_info, double huber_a, const double *pose7,
                           double *H36, double *g6, double *cost);

/* ---- PoseLocalParameterization::Plus (pose_local_parameterization.cpp:26-46), V36 may be null. */
int mloam_pose_plus(mloam_ctx_t *ctx, const double *x7, const double *delta6, const double *V36, double *out7);

/* ---- scan2MapOptimization (lidar_mapper_keyframe.cpp:423-639, gf_method wo_gf).  Maps must have been
 * built in slots MLOAM_MAP_SURF / MLOAM_MAP_CORNER.  The scan features are the (already down-sampled)
 * laser_cloud_surf_cov / laser_cloud_corner_cov in the sensor(base) frame. */
int mloam_scan2map(mloam_ctx_t *ctx, const mloam_point_t *h_surf_scan, int n_surf, const mloam_point_t *h_corner_scan,
                   int n_corner, const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats);
int mloam_scan2map_device(mloam_ctx_t *ctx, const mloam_point_t *d_surf_scan, int n_surf,
                          const mloam_point_t *d_corner_scan, int n_corner, const double *pose_init7,
                          double *pose_out7, mloam_solve_stats_t *stats);

/* ---- uncertainty-aware mapping (with_ua): evalPointUncertainty (associate_uct.hpp:164-215) for a batch of points
 * under the pose `pose7` with covariance cov_pose36 (row-major 6x6: translation, rotation) and measurement covariance
 * cov_meas9 (COV_MEASUREMENT); h_cov6[n*6] receives PointIWithCov::cov_vec (float xx xy xz yy yz zz).
 * mloam_scan2map_ua is mloam_scan2map with every residual weighted by the clamped sqrt(1/trace) of its scan point's
 * covariance (extractCov + lidar_map_factor.hpp:34,41; lidar_mapper_keyframe.cpp:541-545,556-560). */
int mloam_point_uncertainty(mloam_ctx_t *ctx, const mloam_point_t *h_pts, int n, const double *pose7, const double *cov_pose36,
                            const double *cov_meas9, float *h_cov6);
int mloam_scan2map_ua(mloam_ctx_t *ctx, const mloam_point_t *h_surf_scan, int n_surf, const float *h_surf_cov6,
                      const mloam_point_t *h_corner_scan, int n_corner, const float *h_corner_cov6, const double *pose_init7,
                      double *pose_out7, mloam_solve_stats_t *stats);

/* ---- submap assembly with uncertainty: the data path of extractSurroundingKeyFrames (lidar_mapper_keyframe.cpp:254-354).
 * Pose covariances are row-major 6x6 in the reference's order [translation | rotation].
 * mloam_compound_pose_cov: compoundPoseWithCov (associate_uct.hpp:9-88, method 2), host-side: pose_out = pose1 * pose2 with its covariance.
 * mloam_cloud_uct_associate: cloudUCTAssociateToMap (:1116-1158) for one keyframe cloud (intensity = laser id): per point
 *   pose_ext[id]^-1 -> evalPointUncertainty under pose_compound[id] / cov_compound[id] (= compoundPoseWithCov(pose_global, pose_ext[id]))
 *   -> dropped when trace > trace_threshold (TRACE_THRESHOLD_MAPPING) -> pointAssociateToMap with pose_global -> updateCov.  with_ua = 0:
 *   no gate, zero covariance.  Outputs (capacity n): points, cov_vec (xx xy xz yy yz zz), cov_trace, in input order.
 * mloam_voxel_downsample_cov: VoxelGridCovarianceMLOAM<PointIWithCov>::filter — the covariance-weighted merge per voxel
 *   (voxel_grid_covariance_mloam_impl.hpp:293-333): w = trace_threshold - trace, points with |trace| >= trace_threshold skipped.
 * mloam_submap_assemble: n_keyframes clouds (concatenated, counts[k] points each) -> cloudUCTAssociateToMap with poses7[k] and the
 *   per-(keyframe, LiDAR) compounds (pose_compound7 / cov_compound36: n_keyframes x n_lasers) -> merged -> VoxelGridCovarianceMLOAM(leaf,
 *   trace_threshold_filter) -> installed in map slot `slot` (setInputCloud) without leaving the device.  h_out / h_cov6_out (nullable,
 *   capacity = sum of counts) receive the submap; *n_out its size. */
int mloam_compound_pose_cov(const double *pose1_7, const double *cov1_36, const double *pose2_7, const double *cov2_36, double *pose_out7,
                            double *cov_out36);
int mloam_cloud_uct_associate(mloam_ctx_t *ctx, const mloam_point_t *h_pts, int n, const double *pose_global7, int n_lasers, const double *ext7,
                              const double *pose_compound7, const double *cov_compound36, const double *cov_meas9, int with_ua,
                              double trace_threshold, mloam_point_t *h_out, float *h_cov6_out, float *h_trace_out, int *n_out);
int mloam_voxel_downsample_cov(mloam_ctx_t *ctx, const mloam_point_t *h_pts, const float *h_cov6, const float *h_trace, int n, float leaf,
                               float trace_threshold, mloam_point_t *h_out, float *h_cov6_out, float *h_trace_out, int *n_out);
int mloam_submap_assemble(mloam_ctx_t *ctx, int slot, int n_keyframes, const mloam_point_t *h_pts, const int *counts, const double *poses7,
                          int n_lasers, const double *ext7, const double *pose_compound7, const double *cov_compound36, const double *cov_meas9,
                          int with_ua, double trace_threshold_assoc, float leaf, float trace_threshold_filter, float map_cell,
                          mloam_point_t *h_out, float *h_cov6_out, int *n_out);

/* ---- the whole per-scan hot path for one LiDAR sweep (extractCloud -> scan down-sampling ->
 * scan2MapOptimization), inputs in host memory (mloam_frame) or already resident in HBM
 * (mloam_frame_device).  rebuild_maps != 0 re-runs setInputCloud on the two maps first, as the reference
 * does every frame (lidar_mapper_keyframe.cpp:433-434). */
int mloam_frame(mloam_ctx_t *ctx, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end,
                int n_scans, const mloam_point_t *h_surf_map, int n_surf_map, const mloam_point_t *h_corner_map,
                int n_corner_map, int rebuild_maps, const double *pose_init7, double *pose_out7,
                mloam_solve_stats_t *stats);

/* ---- sweep look-ahead.  Announce the sweep of the NEXT mloam_frame / mloam_frame_device call: while the coming frame is matched and
 *      solved, the announced sweep is extracted and down-sampled on a side stream, so that the next call starts at the matching.  The
 *      reference overlaps the same two stages by running them in different nodes (estimator: estimator.cpp:249-263 -> lidar_mapper:
 *      lidar_mapper_keyframe.cpp:356-596).  The next call must pass the SAME pointer and sizes to pick the features up; any other call
 *      extracts as usual.  Poses and statistics are identical with and without announcements.  n <= 0 withdraws.  Host variant: the
 *      buffers must stay valid until the coming frame call returns. */
int mloam_frame_set_next(mloam_ctx_t *ctx, const mloam_point_t *h_cloud, int n, const int *h_scan_start, const int *h_scan_end, int n_scans);
int mloam_frame_set_next_device(mloam_ctx_t *ctx, const mloam_point_t *d_cloud, int n, const int *d_scan_start, const int *d_scan_end,
                                int n_scans);
int mloam_frame_device(mloam_ctx_t *ctx, const mloam_point_t *d_cloud, int n, const int *d_scan_start,
                       const int *d_scan_end, int n_scans, const mloam_point_t *d_surf_map, int n_surf_map,
                       const mloam_point_t *d_corner_map, int n_corner_map, int rebuild_maps,
                       const double *pose_init7, double *pose_out7, mloam_solve_stats_t *stats);

/* Extrinsic of this context's LiDAR (sensor -> base), applied to the extracted features before scan down-sampling
 * and matching in mloam_frame*, as the odometry node does before handing features to the mapper
 * (features reach scan2MapOptimization in the base frame, laser id in intensity; visualization.cpp:48,94-100).
 * NULL resets to identity (no transform). */
int mloam_set_extrinsic(mloam_ctx_t *ctx, const double *ext7);
/* Several LiDARs in ONE context (one GPU): mloam_frame* then takes the sweeps of all n_lidars LiDARs concatenated
 * (LiDAR-major; n_scans = n_lidars x rings per LiDAR, scan_start / scan_end index the concatenation).  extractCloud runs as one
 * batch over all rings (estimator.cpp:249-263 runs it per LiDAR under OpenMP), every LiDAR's features are moved to the base
 * frame with its extrinsic ext7[l] (sensor -> base) and tagged intensity = l (transformCloudFeature, visualization.cpp:40-52),
 * concatenated LiDAR by LiDAR (pubPointCloud, :93-104) and enter downsampleCurrentScan + scan2MapOptimization as ONE feature list
 * (lidar_mapper_keyframe.cpp:356-639).  n_lidars = 1 restores the single-LiDAR path. */
int mloam_set_lidars(mloam_ctx_t *ctx, int n_lidars, const double *ext7);

/* ---- uncertainty-aware mapping (with_ua) in mloam_frame*: the configuration every mapper launch file of the reference runs
 *      (the launch files under estimator/launch set -with_ua=true).
 * mloam_set_uncertainty: with_ua != 0 turns the with_ua branches of the frame on; 0 restores the with_ua = false path exactly.
 *   ext_cov36: per LiDAR of the context (n_lidars after mloam_set_lidars, one in the single-LiDAR path) the row-major 6x6 covariance
 *   [translation | rotation] of its extrinsic, pose_ext[l].cov_, as the /extrinsics message delivers it every frame
 *   (lidar_mapper_keyframe.cpp:1043); cov_meas9 = COV_MEASUREMENT; trace_threshold = TRACE_THRESHOLD_MAPPING.  May be called before
 *   every frame: the values are staged, a captured frame replays with them.  Call it after mloam_set_lidars.  A context with a
 *   communicator (mloam_comm_init / mloam_comm_p2p_init) rejects with_ua frames with MLOAM_E_STATE.
 *   With with_ua, a frame runs downsampleCurrentScan's uncertainty loop (:356-421) after the scan filters: per point
 *   idx = int(intensity) (the laser id of the rig merge; 0 in the single-LiDAR path without mloam_set_lidars extrinsics),
 *   pointAssociateToMap with pose_ext[idx]^-1, evalPointUncertainty under pose_ext[idx] (associate_uct.hpp:196-215), dropped when
 *   trace > TRACE_THRESHOLD_MAPPING; every residual is weighted by sqrt_info of its point's covariance (extractCov + clamp, :541-560,
 *   lidar_map_factor.hpp:34,41), good-feature selection included (lidar_mapper.h:130-174); stats->n_*_in count the gated scans.
 * mloam_pose_covariance: pose_wmap_curr.cov_ (:632) of the last mloam_frame* / mloam_scan2map* solve: cov_mapping = H^-1 with H the
 *   loss-corrected J^T J evaluated at the pose the last Solve returned, with the last association (:600-610), inverted by partial-pivot
 *   LU as Eigen's 6x6 inverse.  mloam_scan2map_ua counts as with_ua.  Zeros without with_ua (:621), when the map gate rejected the
 *   frame (:637) and when the last evaluation had no residual rows (Eigen would return inf / NaN there).  The rule "zero while there
 *   are <= 10 keyframes" (:607-608) is the caller's, which knows the keyframe count — or the keyframe store's, when
 *   mloam_keyframe_save takes the covariance itself (cov36 = NULL).
 * mloam_frame_scan: the down-sampled (and, with with_ua, gated) scans of the last mloam_frame* call in the base frame with their
 *   PointIWithCov::cov_vec (float xx xy xz yy yz zz; zeros without with_ua) — laser_cloud_{surf,corner}_cov, what saveKeyframe stores
 *   (:671-677) and mloam_submap_assemble later takes.  Outputs are nullable; capacities in points.  MLOAM_E_STATE before any frame. */
int mloam_set_uncertainty(mloam_ctx_t *ctx, int with_ua, const double *ext_cov36, const double *cov_meas9, double trace_threshold);
int mloam_pose_covariance(mloam_ctx_t *ctx, double *cov36);
int mloam_frame_scan(mloam_ctx_t *ctx, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf, int *n_surf, mloam_point_t *h_corner,
                     float *h_corner_cov6, int cap_corner, int *n_corner);

/* ---- the mapper's keyframe store, kept on the device: saveKeyframe -> clearCloud -> extractSurroundingKeyFrames
 *      (lidar_mapper_keyframe.cpp:641-683, :921-927 at :1101, :254-354).  The mapper loop of process() (:1062-1101) becomes
 *        mloam_set_lidars / mloam_set_uncertainty (the frame's /extrinsics, :1028-1046, read BEFORE the submap as the reference does:
 *        a keyframe entering the surrounding set is associated with the values in effect at the mloam_keyframe_submap call);
 *        pred = pose_wmap_wodom * pose_wodom_curr;  mloam_keyframe_submap(pred);  mloam_frame(..., rebuild_maps = 0, pred);
 *        mloam_keyframe_save(NULL, NULL);  pose_wmap_wodom = pose_out * pose_wodom_curr^-1
 *      and no point of a keyframe crosses PCIe.  Single-GPU: a context with a communicator gets MLOAM_E_STATE.
 * mloam_keyframes_init: an empty store (DISTANCE_KEYFRAMES [m], ORIENTATION_KEYFRAMES [deg], SURROUNDING_KF_RADIUS [m], MAP_SUR_KF_RES [m],
 *   TRACE_THRESHOLD_MAPPING for the submap association gate and both map filters) and empty map slots MLOAM_MAP_SURF / MLOAM_MAP_CORNER,
 *   so that the first frames fail the map gate (:429).  The map filters use params.surf_leaf / corner_leaf (MAP_SURF_RES / MAP_CORNER_RES,
 *   the leaves of the scan filters too, :1278-1289).
 * mloam_keyframe_save: saveKeyframe for the last mloam_frame* call.  Saved when it is the first keyframe, the float distance of the positions
 *   to the previous keyframe is > DISTANCE_KEYFRAMES, or Eigen's angularDistance 2 atan2(|(q q_prev^-1).vec|, |(q q_prev^-1).w|) in degrees
 *   is > ORIENTATION_KEYFRAMES.  A saved keyframe keeps the frame's down-sampled, gated scans (as mloam_frame_scan returns them), copied
 *   device to device, and marks the submap stale (clearCloud).  pose7 / cov36 NULL: the frame's pose and mloam_pose_covariance, zeroed
 *   while the store holds <= 10 keyframes (:607-608; the count before this save is the one the solve saw); explicit values let a caller
 *   correct keyframe poses.  *saved (nullable) = 1 when saved.  MLOAM_E_STATE if no frame has run since the last save or init.
 * mloam_keyframe_submap: extractSurroundingKeyFrames at the frame's initial guess pose_pred7 (transformAssociateToMap).  Nothing to do
 *   without keyframes, or while both filtered maps hold points (the reference rebuilds while either is empty).  Otherwise: the keyframes
 *   with float squared distance d2 < radius^2 of the prediction, ascending (d2, id); ids that left the set are dropped, survivors keep
 *   their order, new ids are appended in radius order; a new id's clouds are associated ONCE (cloudUCTAssociateToMap with its pose and
 *   covariance and the extrinsics / covariances of mloam_set_lidars / mloam_set_uncertainty at that moment) and cached on the device while
 *   it stays in the set; the set's positions go through VoxelGridCovarianceMLOAM<PointI>(MAP_SUR_KF_RES) with intensity = position in the
 *   set (the last one per voxel wins); the chosen cached clouds are appended in filter order to the merged clouds (emptied by a save only),
 *   filtered with VoxelGridCovarianceMLOAM<PointIWithCov> and built into the two map slots.  *rebuilt (nullable) = 1 when it rebuilt.
 *   *n_surf / *n_corner: the current map sizes; h_* (nullable, capacities in points) receive the maps and their cov_vec.
 * mloam_keyframe_query: keyframe count, surrounding_existing_keyframes_id in order, the keyframe ids the position filter chose in the last
 *   rebuild (filter order).  Outputs nullable.
 * mloam_keyframe_scan: keyframe `id`'s pose, covariance and stored scans (points + cov_vec; outputs nullable, capacities in points). */
int mloam_keyframes_init(mloam_ctx_t *ctx, double distance_keyframes, double orientation_keyframes_deg, double surrounding_kf_radius,
                         double map_sur_kf_res, double trace_threshold);
int mloam_keyframe_save(mloam_ctx_t *ctx, const double *pose7, const double *cov36, int *saved);
int mloam_keyframe_submap(mloam_ctx_t *ctx, const double *pose_pred7, int *rebuilt, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf,
                          int *n_surf, mloam_point_t *h_corner, float *h_corner_cov6, int cap_corner, int *n_corner);
int mloam_keyframe_query(mloam_ctx_t *ctx, int *n_keyframes, int *h_surrounding, int cap_surrounding, int *n_surrounding, int *h_chosen,
                         int cap_chosen, int *n_chosen);
int mloam_keyframe_scan(mloam_ctx_t *ctx, int id, double *pose7, double *cov36, mloam_point_t *h_surf, float *h_surf_cov6, int cap_surf,
                        int *n_surf, mloam_point_t *h_corner, float *h_corner_cov6, int cap_corner, int *n_corner);

/* ---- FeatureExtract::matchCornerFromScan / matchSurfFromScan (feature_extract.hpp:131-376) against the map slot
 * built (mloam_map_build, cell ~1.3 m) from the previous sweep's less-sharp / less-flat features, which must be in
 * the reference's ring-sorted order (int(intensity) = ring).  type 'c': coeffs = [X_closest; X_second];
 * 's': (w, d, 0, 0).  nn3 (nullable): [closest, ind2, ind3] per query (-1 when absent). */
int mloam_match_from_scan(mloam_ctx_t *ctx, int slot, int type, const mloam_point_t *h_pts, int n, const double *pose7,
                          unsigned char *h_valid, double *h_coeffs, int *h_nn3);

/* ---- LidarTracker::trackCloud (lidar_tracker.cpp:23-129). */
int mloam_track_cloud(mloam_ctx_t *ctx, const mloam_point_t *h_prev_less_sharp, int n_pls,
                      const mloam_point_t *h_prev_less_flat, int n_plf, const mloam_point_t *h_cur_sharp, int n_cs,
                      const mloam_point_t *h_cur_flat, int n_cf, const double *pose_ini7, double *pose_out7,
                      mloam_solve_stats_t *stats);

/* ---- Estimator::optimizeMap's LiDAR residual blocks for one frame i / one LiDAR n (estimator.cpp:687-848):
 * LidarPureOdom{PlaneNorm,Edge}Factor (lidar_pure_odom_factor.hpp:27-381) on (pose_pivot [constant, :631], pose_i, ext_n),
 * ceres::HuberLoss(huber_a = 1.0, :602), ceres::Solve(DENSE_SCHUR, max_iterations = NUM_ITERATIONS, :605-615).
 * free_mask: 1 = pose_i free (1x6 odometry rows, ext constant as with ESTIMATE_EXTRINSIC == 0, :640), 2 = ext free
 * (1x6), 3 = both free (1x12 calibration rows [J_pose_i | J_ext], 12x12 normal equations).
 * Features are the matcher's output (types[n] 's'|'c', sensor-frame points n*3, coefficients n*6 in the pivot frame).
 * pose_i7 / ext7 are updated in place.  stats->H receives the leading 6x6 block of J^T J. */
int mloam_odom_solve(mloam_ctx_t *ctx, int n, const unsigned char *h_types, const double *h_points, const double *h_coeffs,
                     const double *pose_pivot7, double *pose_i7, double *ext7, int free_mask, int max_iterations,
                     double huber_a, double sqrt_info, mloam_solve_stats_t *stats);

/* ---- online extrinsic calibration step: Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 (estimator.cpp:687-787) for one frame i
 * and one calibrated LiDAR, with the association of buildCalibMap (:1067-1156) redone at every outer iteration.
 * State [pose_i | ext_cal] (12-DoF); pose_pivot and ext_ref are constant blocks (:631, :642).
 *   reference LiDAR, frame i : features (sensor frame) are matched at pivot^-1 * pose_i * ext_ref against the local map in slots
 *     MLOAM_MAP_CORNER / MLOAM_MAP_SURF with n_neigh = 5, CHECK_FOV = true (:1135-1149) and enter as LidarPureOdom{PlaneNorm,Edge}Factor
 *     on (pivot, pose_i, ext_ref) — 1x6 rows on pose_i;
 *   calibrated LiDAR, pivot frame : features are matched at ext_cal (n_neigh = 10, CHECK_FOV = true) against slots
 *     MLOAM_MAP_SCAN_CORNER / MLOAM_MAP_SCAN_SURF when own_cal_maps != 0 (its own local map, leaf 0.2, :1103-1109), else the same maps,
 *     and enter as LidarOnlineCalib{PlaneNorm,Edge}Factor on ext_cal (lidar_online_calib_factor.hpp:24-227) — 1x6 rows on ext_cal.
 * Either group may be empty: with a communicator (mloam_comm_init) rank 0 passes the reference LiDAR's features, rank 1 the
 * calibrated LiDAR's, and the packed 12x12 normal equations (92 doubles) are summed with one ncclAllReduce per LM evaluation
 * (SURVEY.md 8e); every rank applies the identical step.  ceres::Solve: max_outer x (re-association + <= max_inner LM iterations),
 * HuberLoss(huber_a = 1.0, :602).  stats->n_surf = residual rows of the last evaluation (all ranks), stats->H = the pose block. */
int mloam_calib_frame(mloam_ctx_t *ctx, const mloam_point_t *h_surf_ref, int n_surf_ref, const mloam_point_t *h_corner_ref,
                      int n_corner_ref, const mloam_point_t *h_surf_cal, int n_surf_cal, const mloam_point_t *h_corner_cal,
                      int n_corner_cal, const double *pose_pivot7, double *pose_i7, const double *ext_ref7, double *ext_cal7,
                      int max_outer, int max_inner, double huber_a, int own_cal_maps, mloam_solve_stats_t *stats);

/* ---- ActiveFeatureSelection::goodFeatureMatching for one feature set (lidar_mapper.h:229-573; Estimator::goodFeatureMatching,
 * estimator.cpp:1347-1517): match every feature of `h_pts` against map `slot` at pose7, evaluate its 1x6 Jacobian row
 * (evaluateFeatJacobianMatching, lidar_mapper.h:130-174; sqrt_info from the point's covariance h_cov6[n*6] — PointIWithCov::cov_vec —
 * or from params.cov_trace when null) and select gf_ratio * n features.
 * method: 0 wo_gf (all matched), 1 rnd, 2 fps, 3 gd_fix / gd_float (stochastic greedy on log det(H + J^T J)).
 * The reference's mt19937(random_device) becomes an explicit PCG32 `seed` and its wall-clock cap (MAX_FEATURE_SELECT_TIME)
 * is dropped; MAX_RANDOM_QUEUE_TIME = 20 is kept.  Outputs: h_sel[<= n] feature indices in selection order, *n_sel,
 * H36 = sub_mat_H (starts at 1e-6 I), optional h_matched[n] and h_jaco[n*6]. */
int mloam_good_features(mloam_ctx_t *ctx, int slot, int type, const mloam_point_t *h_pts, int n, const float *h_cov6,
                        const double *pose7, int method, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel,
                        double *H36, unsigned char *h_matched, double *h_jaco);

/* ---- Estimator::goodFeatureMatching, the odometry-side twin (estimator.cpp:1347-1517): features of frame i (sensor frame) against the local map
 * in `slot`, matched at pose_local = pivot^-1 * pose_i * ext (n_neigh 5, CHECK_FOV false); rows from evaluateFeatJacobian (:1273-1345):
 * surf -> the pose_i block of LidarPureOdomPlaneNormFactor(point, coeffs, 1.0), corner -> the constant row [1 0 0 0 0 0] (:1342).
 * gf_ratio == 1.0: every matched feature in order (:1380-1414); else the stochastic greedy selection (seed instead of random_device, no
 * wall-clock cap).  Outputs as mloam_good_features. */
int mloam_good_features_odom(mloam_ctx_t *ctx, int slot, int type, const mloam_point_t *h_pts, int n, const double *pose_pivot7,
                             const double *pose_i7, const double *ext7, double gf_ratio, unsigned long long seed, int *h_sel, int *n_sel,
                             double *H36, unsigned char *h_matched, double *h_jaco);

/* ---- Estimator::buildLocalMap / buildCalibMap, the map half (estimator.cpp:1175-1204 / :1084-1110) for one LiDAR and one feature kind:
 * the window's stacked clouds (n_frames clouds concatenated, counts[i] points each, sensor frame) are moved into the pivot frame with
 * pose_local7[i] = pivot^-1 * pose_i * ext (pcl::transformPointCloud with the float matrix, intensity kept), concatenated,
 * filtered with pcl::VoxelGrid(leaf) (leaf = 0.4 * clamp(N_SCANS * NUM_OF_LASER * WINDOW_SIZE / 192, 0.75, 2) in buildLocalMap :1194;
 * 0.4 / 0.2 in buildCalibMap :1103) and installed in map slot `slot` (setInputCloud, :1231-1233).  h_out (nullable, capacity = sum of
 * counts) receives the filtered local map, *n_out its size.  The frames of the window are then matched with mloam_match_from_map /
 * mloam_good_features_odom and solved with mloam_odom_solve / mloam_calib_frame. */
int mloam_local_map_build(mloam_ctx_t *ctx, int slot, int n_frames, const mloam_point_t *h_pts, const int *counts, const double *pose_local7,
                          float leaf, float map_cell, mloam_point_t *h_out, int *n_out);

/* ---- multi-GPU: one LiDAR per GPU, one all-reduce of the packed normal equations per LM evaluation
 * (SURVEY.md §8e).  id128 is an ncclUniqueId (128 bytes) created on rank 0 and shared by the caller. */
int mloam_comm_unique_id(void *id128);
int mloam_comm_init(mloam_ctx_t *ctx, int nranks, int rank, const void *id128);
int mloam_comm_destroy(mloam_ctx_t *ctx);
/* Peer-memory exchange: when every GPU of the node can map every other (NVLink / NVSwitch), the all-reduce, the
 * partial-sum kernel before it and the LM-step kernel after it collapse into the tail of the residual kernel: each
 * rank stores its 30 packed doubles into every rank's exchange buffer, raises a flag, polls its own buffer and sums
 * the contributions in rank order.  export: create this rank's buffer, return its cudaIpcMemHandle_t (64 bytes);
 * init: handles = nranks x 64 bytes gathered by the caller (rank order).  Falls back to NCCL when not initialised. */
int mloam_comm_p2p_export(mloam_ctx_t *ctx, void *handle64);
int mloam_comm_p2p_init(mloam_ctx_t *ctx, int nranks, int rank, const void *handles);
/* The exchange is collective: every rank must run the same sequence of mloam_frame* / mloam_scan2map* calls (the map-size gate
 * depends on the replicated maps only).  Solves that belong to one rank alone (mloam_track_cloud, mloam_odom_solve,
 * mloam_normal_equations) never exchange.  A rank that waits ~3 s for a peer, or finds a peer AHEAD of the exchange it expects
 * (lost lock-step), ends the solve with termination 9 and the call returns MLOAM_E_NCCL on that rank; recover by calling
 * mloam_comm_p2p_reset on every rank between two host-side barriers. */
int mloam_comm_p2p_reset(mloam_ctx_t *ctx);

#ifdef __cplusplus
}
#endif
#endif /* MLOAM_B200_H_ */
