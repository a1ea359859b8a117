// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The mapper's keyframe state machine of lidar_mapper_keyframe.cpp as a stateful restatement for tests/mapper_lib.py (liborc_mapper.so,
// built from orc_ua.cpp + the same headers):
//   saveKeyframe                  :641-683 (Mapper::save)
//   clearCloud                    :921-927, called after a save (:1101)
//   extractSurroundingKeyFrames   :254-354 (Mapper::submap): radius search, the surrounding-set bookkeeping (:274-323) with the cached
//                                 associated clouds, the keyframe-position filter (:325-338), `+=` and the two covariance filters (:339-347)
//   process()                     :1062-1101 (orc_mapper_process): transformAssociateToMap -> extractSurroundingKeyFrames ->
//                                 downsampleCurrentScan + scan2MapOptimization (orc_ua_frame_multi / orc::scan2map) -> transformUpdate ->
//                                 saveKeyframe (-> clearCloud)
// Restatement choices (in addition to orc_math.hpp's and orc_ua.cpp's):
//   - the distance test of saveKeyframe is evaluated in float (pose_point_cur / pose_point_prev are PointI): float differences, the float
//     sum of their squares left to right, sqrtf, compared as double with DISTANCE_KEYFRAMES;
//   - angularDistance is Eigen's 2 atan2(|d.vec|, |d.w|), d = q_cur * conj(q_prev), |d.vec| = sqrt((x*x + y*y) + z*z);
//   - the radius search (pcl::KdTreeFLANN over pose_keyframes_3d; the reference does not vendor FLANN) keeps keyframes with the float
//     L2_Simple distance d2 = ((0 + dx*dx) + dy*dy) + dz*dz strictly below (float)(radius * radius) — FLANN's RadiusResultSet adds a
//     point when dist < radius — and orders them by (d2, keyframe id);
//   - the keyframe pose and the extrinsics enter compoundPoseWithCov normalised, as mloam_compound_pose_cov takes them; the keyframe
//     pose moves the points as given (pointAssociateToMap).
#include "orc_ua.cpp"

namespace {

struct Keyframe {
  double pose[7], cov[36];
  PointI pos;  // pose_keyframes_3d, intensity = id
  Cloud surf, corner;
};

struct Mapper {
  double dist_kf, orient_deg, radius, trace_thr;
  float sur_kf_res, surf_leaf, corner_leaf;
  int n_lasers = 1, with_ua = 0;
  std::vector<double> ext7, ext_cov36;
  double cov_meas[9] = {0};
  PointI prev_pt{0.f, 0.f, 0.f, 0.f};
  Q4 prev_q{0, 0, 0, 1};
  std::vector<Keyframe> kfs;
  std::vector<int> sur_ids;                   // surrounding_existing_keyframes_id
  std::vector<CovCloud> sur_surf, sur_corner;  // surrounding_{surf,corner}_cloud_keyframes
  CovCloud surf_raw, corner_raw;              // laser_cloud_{surf,corner}_from_map_cov
  CovCloud surf_ds, corner_ds;                // laser_cloud_{surf,corner}_from_map_cov_ds
  std::vector<int> chosen;
  double last_margin[2] = {0, 0};  // saveKeyframe: distance - DISTANCE_KEYFRAMES [m], angle - ORIENTATION_KEYFRAMES [deg]
  double radius_margin = 1e30;     // min |d2 - radius^2| of the last radius search
  Pose wmap_wodom;                 // pose_wmap_wodom (identity)

  // saveKeyframe (:641-683); returns save_new_keyframe
  bool save(const double *pose7, const double *cov36, const Cloud &surf, const Cloud &corner) {
    const PointI cur{(float)pose7[0], (float)pose7[1], (float)pose7[2], 0.f};
    const float dx = cur.x - prev_pt.x, dy = cur.y - prev_pt.y, dz = cur.z - prev_pt.z;
    const float dist = sqrtf(dx * dx + dy * dy + dz * dz);
    const Q4 d = qmul(Q4{pose7[3], pose7[4], pose7[5], pose7[6]}, qconj(prev_q));
    const double ang = 2.0 * std::atan2(std::sqrt(d.x * d.x + d.y * d.y + d.z * d.z), std::fabs(d.w)) / 3.14159265358979323846 * 180.0;  // / M_PI * 180
    last_margin[0] = (double)dist - dist_kf, last_margin[1] = ang - orient_deg;
    if (!((double)dist > dist_kf || ang > orient_deg || kfs.empty())) return false;
    prev_pt = cur, prev_q = Q4{pose7[3], pose7[4], pose7[5], pose7[6]};
    Keyframe k;
    std::memcpy(k.pose, pose7, sizeof(k.pose)), std::memcpy(k.cov, cov36, sizeof(k.cov));
    k.pos = PointI{cur.x, cur.y, cur.z, (float)kfs.size()};
    k.surf = surf, k.corner = corner;
    kfs.push_back(k);
    clear_cloud();
    return true;
  }
  // clearCloud (:921-927)
  void clear_cloud() {
    for (CovCloud *c : {&surf_raw, &corner_raw, &surf_ds, &corner_ds}) c->pts.clear(), c->cov6.clear(), c->trace.clear();
  }
  // cloudUCTAssociateToMap (:1116-1158) of one keyframe with the current extrinsics and covariances
  void associate_kf(const Keyframe &k, const Cloud &in, CovCloud &out) const {
    std::vector<Pose> pe, pc;
    std::vector<M6> cc(n_lasers);
    M6 kc;
    std::memcpy(kc.m, k.cov, sizeof(kc.m));
    for (int l = 0; l < n_lasers; l++) {
      const double *e = &ext7[7 * (size_t)l];
      pe.push_back(to_pose(e));
      M6 ec;
      for (int q = 0; q < 36; q++) ec.m[q] = with_ua ? ext_cov36[36 * (size_t)l + q] : 0.0;
      Pose p;
      compound_pose_with_cov(make_pose(Q4{k.pose[3], k.pose[4], k.pose[5], k.pose[6]}, V3{k.pose[0], k.pose[1], k.pose[2]}), kc,
                             make_pose(Q4{e[3], e[4], e[5], e[6]}, V3{e[0], e[1], e[2]}), ec, p, cc[l]);
      pc.push_back(p);
    }
    cloud_uct_associate(in, to_pose(k.pose), pe, pc, cc, cov_meas, with_ua != 0, trace_thr, out);
  }
  // extractSurroundingKeyFrames (:254-354); returns whether it rebuilt the maps
  bool submap(const double *pred7) {
    if (kfs.empty()) return false;                                                   // :256
    if (!surf_ds.pts.empty() && !corner_ds.pts.empty()) return false;                // :257
    const PointI q{(float)pred7[0], (float)pred7[1], (float)pred7[2], 0.f};          // :264-266
    const float r2 = (float)(radius * radius);
    std::vector<std::pair<float, int>> found;                                        // :268-272
    radius_margin = 1e30;
    for (const Keyframe &k : kfs) {
      float d2 = 0.f;
      const float a = k.pos.x - q.x, b = k.pos.y - q.y, c = k.pos.z - q.z;
      d2 += a * a, d2 += b * b, d2 += c * c;
      radius_margin = std::min(radius_margin, std::fabs((double)d2 - (double)r2));
      if (d2 < r2) found.push_back({d2, (int)k.pos.intensity});
    }
    std::sort(found.begin(), found.end());
    for (int i = 0; i < (int)sur_ids.size(); i++) {                                  // :274-292
      bool existing = false;
      for (const auto &f : found)
        if (sur_ids[i] == f.second) {
          existing = true;
          break;
        }
      if (!existing) {
        sur_ids.erase(sur_ids.begin() + i), sur_surf.erase(sur_surf.begin() + i), sur_corner.erase(sur_corner.begin() + i);
        i--;
      }
    }
    for (const auto &f : found) {                                                    // :294-323
      bool existing = false;
      for (int id : sur_ids)
        if (id == f.second) {
          existing = true;
          break;
        }
      if (existing) continue;
      sur_ids.push_back(f.second);
      CovCloud s, c;
      associate_kf(kfs[f.second], kfs[f.second].surf, s);
      associate_kf(kfs[f.second], kfs[f.second].corner, c);
      sur_surf.push_back(s), sur_corner.push_back(c);
    }
    Cloud pos, pos_ds;                                                               // :325-335
    for (int i = 0; i < (int)sur_ids.size(); i++) {
      PointI p = kfs[sur_ids[i]].pos;
      p.intensity = (float)i;
      pos.push_back(p);
    }
    voxel_grid(pos, sur_kf_res, pos_ds, true);
    chosen.clear();
    auto append = [](CovCloud &dst, const CovCloud &src) {
      dst.pts.insert(dst.pts.end(), src.pts.begin(), src.pts.end());
      dst.cov6.insert(dst.cov6.end(), src.cov6.begin(), src.cov6.end());
      dst.trace.insert(dst.trace.end(), src.trace.begin(), src.trace.end());
    };
    for (const PointI &p : pos_ds) {                                                 // :336-341
      const int j = (int)p.intensity;
      chosen.push_back(sur_ids[j]);
      append(surf_raw, sur_surf[j]), append(corner_raw, sur_corner[j]);
    }
    voxel_grid_cov(surf_raw, surf_leaf, (float)trace_thr, surf_ds);                  // :344-347
    voxel_grid_cov(corner_raw, corner_leaf, (float)trace_thr, corner_ds);
    return true;
  }
  // kept entries whose association under the CURRENT extrinsic covariances would differ from the cached one (the cache decides)
  int reassoc_differs() const {
    int n = 0;
    for (size_t i = 0; i < sur_ids.size(); i++) {
      CovCloud s;
      associate_kf(kfs[sur_ids[i]], kfs[sur_ids[i]].surf, s);
      const CovCloud &o = sur_surf[i];
      if (s.pts.size() != o.pts.size() || std::memcmp(s.pts.data(), o.pts.data(), sizeof(PointI) * s.pts.size()) != 0 ||
          std::memcmp(s.cov6.data(), o.cov6.data(), sizeof(float) * s.cov6.size()) != 0)
        n++;
    }
    return n;
  }
};

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

// saveKeyframe with the given pose, covariance and scans; margins2 (nullable): distance and angle minus their thresholds
int orc_mapper_save(void *h, const double *pose7, const double *cov36, const float *surf, int n_surf, const float *corner, int n_corner,
                    double *margins2) {
  Mapper *m = static_cast<Mapper *>(h);
  const bool s = m->save(pose7, cov36, cloud_of(surf, n_surf), cloud_of(corner, n_corner));
  if (margins2) margins2[0] = m->last_margin[0], margins2[1] = m->last_margin[1];
  return s ? 1 : 0;
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

// ---- one pass of process() (:1062-1101) over a rig sweep (the inputs of orc_ua_frame_multi) with the odometry pose odom7:
// pose_wmap_curr = pose_wmap_wodom * odom (transformAssociateToMap, pose.cpp's operator*) -> extractSurroundingKeyFrames -> the frame
// (with_ua: orc_ua_frame_multi with frame_trace_threshold; else the plain frame) against the current maps -> cov_mapping zeroed while
// <= 10 keyframes (:607-608) -> transformUpdate (pose_wmap_wodom = pose_wmap_curr * odom^-1) -> saveKeyframe.
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
  Cloud sm = m->surf_ds.pts, cm = m->corner_ds.pts;
  double stats[20], cov[36];
  std::vector<float> so(4 * (size_t)n), sc(6 * (size_t)n), co(4 * (size_t)n), cc(6 * (size_t)n);
  int ns = 0, nc = 0;
  if (m->with_ua) {
    orc_ua_frame_multi(cloud, n, scan_start, scan_end, n_scans, m->n_lasers, m->ext7.data(), m->ext_cov36.data(), m->cov_meas,
                       frame_trace_threshold, reinterpret_cast<const float *>(sm.data()), (int)sm.size(), reinterpret_cast<const float *>(cm.data()),
                       (int)cm.size(), m->corner_leaf, m->surf_leaf, pred7, opts, pose_out7, stats, cov, nullptr, so.data(), sc.data(), &ns,
                       co.data(), cc.data(), &nc);
  } else {
    Cloud cs, ss;
    prepare_multi(cloud, n, scan_start, scan_end, n_scans, m->n_lasers, m->ext7.data(), m->corner_leaf, m->surf_leaf, cs, ss);
    const Scan2MapResult r = scan2map(sm, cm, ss, cs, pred, opts_from(opts));
    pose_to_param(r.pose, pose_out7);
    stats[1] = r.ran;
    stats[0] = r.ran;
    std::memset(cov, 0, sizeof(cov));
    ns = (int)ss.size(), nc = (int)cs.size();
    std::memcpy(so.data(), ss.data(), sizeof(PointI) * ss.size()), std::memcpy(co.data(), cs.data(), sizeof(PointI) * cs.size());
  }
  std::memcpy(cov36, cov, sizeof(cov));                         // H^-1 of the solve (mloam_pose_covariance)
  if (m->kfs.size() <= 10) std::memset(cov, 0, sizeof(cov));  // cov_mapping as the keyframe keeps it
  const Pose out = to_pose(pose_out7);
  m->wmap_wodom = pose_mul(out, pose_inv(odom));
  const bool saved = m->save(pose_out7, cov, cloud_of(so.data(), ns), cloud_of(co.data(), nc));
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
