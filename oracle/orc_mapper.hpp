// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The mapper's keyframe store (see orc_mapper.cpp), shared by its entry points (orc_mapper.cpp) and the global map (orc_global_map.cpp).
#pragma once
#include "orc_capi.hpp"
#include <algorithm>

namespace orc {

struct Keyframe {
  double pose[7], cov[36];
  PointI pos;  // pose_keyframes_3d, intensity = id
  Cloud surf, corner, outlier;
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

  static void append(CovCloud &dst, const CovCloud &src) {
    dst.pts.insert(dst.pts.end(), src.pts.begin(), src.pts.end());
    dst.cov6.insert(dst.cov6.end(), src.cov6.begin(), src.cov6.end());
    dst.trace.insert(dst.trace.end(), src.trace.begin(), src.trace.end());
  }

  // saveKeyframe (:641-683); returns save_new_keyframe
  bool save(const double *pose7, const double *cov36, const Cloud &surf, const Cloud &corner, const Cloud &outlier) {
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
    k.surf = surf, k.corner = corner, k.outlier = outlier;
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

}  // namespace orc
