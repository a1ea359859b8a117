// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The mapper's keyframe store of lidar_mapper_keyframe.cpp as a stateful restatement (liborc.so's orc_mapper_*; the store is orc_mapper.hpp's
// Mapper, and orc_global_map.cpp builds the global map over it):
//   saveKeyframe                  :641-683 (Mapper::save), with outlier_cloud_keyframes_cov next to surf and corner (:673-681)
//   clearCloud                    :921-927, called after a save (:1101)
//   extractSurroundingKeyFrames   :254-354 (Mapper::submap): radius search, the surrounding-set bookkeeping (:274-323) with the cached
//                                 associated clouds, the keyframe-position filter (:325-338), `+=` and the two covariance filters (:339-347)
//   process()                     :1062-1101 (orc_mapper_process): transformAssociateToMap -> extractSurroundingKeyFrames ->
//                                 downsampleCurrentScan + scan2MapOptimization (frame_ua) -> transformUpdate -> saveKeyframe (-> clearCloud)
// Restatement choices (in addition to orc_math.hpp's and orc_ua.cpp's):
//   - the distance test of saveKeyframe is evaluated in float (pose_point_cur / pose_point_prev are PointI): float differences, the float
//     sum of their squares left to right, sqrtf, compared as double with DISTANCE_KEYFRAMES;
//   - angularDistance is Eigen's 2 atan2(|d.vec|, |d.w|), d = q_cur * conj(q_prev), |d.vec| = sqrt((x*x + y*y) + z*z);
//   - the radius search (pcl::KdTreeFLANN over pose_keyframes_3d; the reference does not vendor FLANN) keeps keyframes with the float
//     L2_Simple distance d2 = ((0 + dx*dx) + dy*dy) + dz*dz strictly below (float)(radius * radius) — FLANN's RadiusResultSet adds a
//     point when dist < radius — and orders them by (d2, keyframe id);
//   - the keyframe pose and the extrinsics enter compoundPoseWithCov normalised, as mloam_compound_pose_cov takes them; the keyframe
//     pose moves the points as given (pointAssociateToMap).
#include "orc_mapper.hpp"

using namespace orc;

namespace {

Cloud cloud_of(const float *p, int n) { return to_cloud(p, n); }

}  // namespace

extern "C" {

void *orc_mapper_create(double distance_keyframes, double orientation_keyframes_deg, double radius, double sur_kf_res, double trace_threshold,
                        float surf_leaf, float corner_leaf) {
  Mapper *m = new Mapper();
  m->dist_kf = distance_keyframes, m->orient_deg = orientation_keyframes_deg, m->radius = radius, m->trace_thr = trace_threshold;
  m->sur_kf_res = (float)sur_kf_res, m->surf_leaf = surf_leaf, m->corner_leaf = corner_leaf;
  return m;
}
void orc_mapper_destroy(void *h) { delete static_cast<Mapper *>(h); }

// pose_ext of the rig (n_lasers x 7), their covariances (n_lasers x 36, the /extrinsics message :1043) and COV_MEASUREMENT; may change
// between frames.  with_ua = 0: cloudUCTAssociateToMap's with_ua_flag = false branch.
void orc_mapper_set_lidars(void *h, int n_lasers, const double *ext7, const double *ext_cov36, const double *cov_meas9, int with_ua) {
  Mapper *m = static_cast<Mapper *>(h);
  m->n_lasers = n_lasers, m->with_ua = with_ua;
  m->ext7.assign(ext7, ext7 + 7 * (size_t)n_lasers);
  m->ext_cov36.assign(36 * (size_t)n_lasers, 0.0);
  if (ext_cov36) m->ext_cov36.assign(ext_cov36, ext_cov36 + 36 * (size_t)n_lasers);
  if (cov_meas9) std::memcpy(m->cov_meas, cov_meas9, sizeof(m->cov_meas));
}

// saveKeyframe with the given pose, covariance and scans; outlier (nullable): the keyframe's outlier cloud (outlier_cloud_keyframes_cov);
// margins2 (nullable): distance and angle minus their thresholds
int orc_mapper_save_outlier(void *h, const double *pose7, const double *cov36, const float *surf, int n_surf, const float *corner, int n_corner,
                            const float *outlier, int n_outlier, double *margins2) {
  Mapper *m = static_cast<Mapper *>(h);
  const bool s = m->save(pose7, cov36, cloud_of(surf, n_surf), cloud_of(corner, n_corner), outlier ? cloud_of(outlier, n_outlier) : Cloud());
  if (margins2) margins2[0] = m->last_margin[0], margins2[1] = m->last_margin[1];
  return s ? 1 : 0;
}
// the same without an outlier cloud
int orc_mapper_save(void *h, const double *pose7, const double *cov36, const float *surf, int n_surf, const float *corner, int n_corner,
                    double *margins2) {
  return orc_mapper_save_outlier(h, pose7, cov36, surf, n_surf, corner, n_corner, nullptr, 0, margins2);
}

// extractSurroundingKeyFrames at pred7; radius_margin (nullable): min |d2 - radius^2| over the keyframes of the last search
int orc_mapper_submap(void *h, const double *pred7, double *radius_margin) {
  Mapper *m = static_cast<Mapper *>(h);
  const bool r = m->submap(pred7);
  if (radius_margin) *radius_margin = r ? m->radius_margin : 1e30;
  return r ? 1 : 0;
}

// counts[5]: keyframes, surrounding ids, chosen ids, surf map, corner map.  Arrays (nullable) sized by a previous call.
void orc_mapper_query(void *h, int *counts, int *sur, int *chosen) {
  const Mapper *m = static_cast<const Mapper *>(h);
  counts[0] = (int)m->kfs.size(), counts[1] = (int)m->sur_ids.size(), counts[2] = (int)m->chosen.size();
  counts[3] = (int)m->surf_ds.pts.size(), counts[4] = (int)m->corner_ds.pts.size();
  if (sur) std::copy(m->sur_ids.begin(), m->sur_ids.end(), sur);
  if (chosen) std::copy(m->chosen.begin(), m->chosen.end(), chosen);
}

// map t (0 surf, 1 corner): points and cov_vec (capacity from orc_mapper_query)
void orc_mapper_map(void *h, int t, float *pts, float *cov6) {
  const Mapper *m = static_cast<const Mapper *>(h);
  const CovCloud &c = t == 0 ? m->surf_ds : m->corner_ds;
  if (!c.pts.empty()) std::memcpy(pts, c.pts.data(), sizeof(PointI) * c.pts.size()), std::memcpy(cov6, c.cov6.data(), sizeof(float) * c.cov6.size());
}

int orc_mapper_reassoc_differs(void *h) { return static_cast<const Mapper *>(h)->reassoc_differs(); }

// pose_keyframes_6d[id]: the pose and covariance saveKeyframe stored
void orc_mapper_keyframe(void *h, int id, double *pose7, double *cov36) {
  const Keyframe &k = static_cast<const Mapper *>(h)->kfs.at((size_t)id);
  std::memcpy(pose7, k.pose, sizeof(k.pose)), std::memcpy(cov36, k.cov, sizeof(k.cov));
}

// ---- one pass of process() (:1062-1101) over a rig sweep (the inputs of orc_frame_ua) with the odometry pose odom7:
// pose_wmap_curr = pose_wmap_wodom * odom (transformAssociateToMap, pose.cpp's operator*) -> extractSurroundingKeyFrames -> the frame
// (frame_ua, with_ua with frame_trace_threshold) against the current maps -> cov_mapping zeroed while <= 10 keyframes (:607-608) ->
// transformUpdate (pose_wmap_wodom = pose_wmap_curr * odom^-1) -> saveKeyframe.
// out: pose_out7, cov36 (H^-1 of the solve, before the <= 10 keyframes rule the saved keyframe gets), info[8] = {rebuilt, ran, saved, distance margin, angle margin, radius margin, n_surf_in, n_corner_in}
void orc_mapper_process(void *h, const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, const double *odom7,
                        double frame_trace_threshold, const double *opts, double *pose_out7, double *cov36, double *info) {
  Mapper *m = static_cast<Mapper *>(h);
  const Pose odom = make_pose(Q4{odom7[3], odom7[4], odom7[5], odom7[6]}, V3{odom7[0], odom7[1], odom7[2]});
  const Pose pred = pose_mul(m->wmap_wodom, odom);
  double pred7[7];
  pose_to_param(pred, pred7);
  double rmarg = 1e30;
  const int rebuilt = orc_mapper_submap(h, pred7, &rmarg);
  const Cloud &sm = m->surf_ds.pts, &cm = m->corner_ds.pts;
  double stats[20], cov[36];
  std::vector<float> so(4 * (size_t)n), co(4 * (size_t)n);
  int ns = 0, nc = 0;
  frame_ua(cloud, n, scan_start, scan_end, n_scans, m->n_lasers, m->ext7.data(), nullptr, nullptr, 0.f, m->with_ua ? m->ext_cov36.data() : nullptr,
           m->cov_meas, frame_trace_threshold, reinterpret_cast<const float *>(sm.data()), (int)sm.size(), reinterpret_cast<const float *>(cm.data()),
           (int)cm.size(), m->corner_leaf, m->surf_leaf, pred7, opts, pose_out7, stats, cov, nullptr, so.data(), nullptr, &ns, co.data(), nullptr, &nc);
  std::memcpy(cov36, cov, sizeof(cov));                         // H^-1 of the solve (mloam_pose_covariance)
  if (m->kfs.size() <= 10) std::memset(cov, 0, sizeof(cov));  // cov_mapping as the keyframe keeps it
  const Pose out = to_pose(pose_out7);
  m->wmap_wodom = pose_mul(out, pose_inv(odom));
  const bool saved = m->save(pose_out7, cov, cloud_of(so.data(), ns), cloud_of(co.data(), nc), Cloud());
  info[0] = rebuilt, info[1] = stats[0], info[2] = saved ? 1 : 0, info[3] = m->last_margin[0], info[4] = m->last_margin[1], info[5] = rmarg;
  info[6] = ns, info[7] = nc;
}

void orc_mapper_pose_mul(const double *a7, const double *b7, double *out7) {
  pose_to_param(pose_mul(make_pose(Q4{a7[3], a7[4], a7[5], a7[6]}, V3{a7[0], a7[1], a7[2]}), make_pose(Q4{b7[3], b7[4], b7[5], b7[6]}, V3{b7[0], b7[1], b7[2]})),
                out7);
}
void orc_mapper_pose_inv(const double *a7, double *out7) {
  pose_to_param(pose_inv(make_pose(Q4{a7[3], a7[4], a7[5], a7[6]}, V3{a7[0], a7[1], a7[2]})), out7);
}

}  // extern "C"
