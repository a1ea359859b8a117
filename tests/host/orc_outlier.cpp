// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/orc_math.hpp's header).
// The outlier cloud of segment_cloud: 0 (laser_cloud_outlier_cov) restated over the oracle's frame and keyframe store (oracle/orc_mapper.cpp,
// included whole, so that the store this library makes is the one its global map reads):
//   ImageSegmenter::segmentCloud       image_segmenter.hpp:390: ONE point per LiDAR, laser_cloud_out.points[0], the first point of its
//                                      ring-ordered cloud; none for an empty cloud (mloam_adapter.hpp:114 skips the undefined read)
//   pubPointCloud / transformCloudFeature  visualization.cpp:40-52, :89-104: pcl::transformPointCloud with Pose(qbl, tbl).T_.cast<float>(),
//                                      intensity = n, concatenated LiDAR by LiDAR
//   downsampleCurrentScan              lidar_mapper_keyframe.cpp:366-368, :407-418: VoxelGridCovarianceMLOAM<PointI>(MAP_OUTLIER_RES)
//                                      (:1283-1284), then with with_ua the scans' gate (pose_ext[idx]^-1, evalPointUncertainty, dropped when
//                                      trace > TRACE_THRESHOLD_MAPPING), cov_vec zero without it
//   saveKeyframe                       :673-681: outlier_cloud_keyframes_cov next to surf and corner
//   pubGlobalMap / saveGlobalMap       :818-827 (surf, corner, outlier into one map) / :873-882 (surf then outlier into the surf map, corner
//                                      into the corner map), each cloud through cloudUCTAssociateToMap under the keyframe's pose
// Restatement choices (in addition to orc_mapper.cpp's and tests/host/orc_global_map.cpp's):
//   - LiDAR l's part of a frame's concatenation is [scan_start[l R] - 5, scan_start[(l + 1) R] - 5) (the last one ends at n), as
//     prepare_multi cuts it;
//   - the store here (OutlierMapper) is orc_mapper.cpp's Mapper plus one outlier cloud per keyframe, appended when Mapper::save saves.
#include "../../oracle/orc_mapper.cpp"

namespace {

// laser_cloud_outlier_cov of one frame
void frame_outlier(const float *cloud, int n, const int *scan_start, int n_scans, int n_lidars, const double *ext7, const double *ext_cov36,
                   const double *cov_meas9, bool with_ua, double trace_threshold, float leaf, Cloud &out, std::vector<float> &cov6) {
  out.clear(), cov6.clear();
  const int R = n_scans / n_lidars;
  Cloud raw;
  for (int l = 0; l < n_lidars; l++) {
    const int lo = scan_start[l * R] - 5, hi = (l + 1 < n_lidars) ? scan_start[(l + 1) * R] - 5 : n;
    if (!(lo < hi) || lo < 0 || lo >= n) continue;  // an empty part pushes no point
    const PointI p = to_cloud(cloud + 4 * (size_t)lo, 1)[0];
    const double *e = ext7 + 7 * l;
    const Pose T = make_pose(Q4{e[3], e[4], e[5], e[6]}, V3{e[0], e[1], e[2]});
    const M3 Rm = qmat(T.q);
    float m[12];
    for (int r = 0; r < 3; r++) {
      for (int k = 0; k < 3; k++) m[4 * r + k] = (float)Rm(r, k);
      m[4 * r + 3] = (float)(r == 0 ? T.t.x : (r == 1 ? T.t.y : T.t.z));
    }
    PointI o;
    o.x = m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3];
    o.y = m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7];
    o.z = m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11];
    o.intensity = (float)l;
    raw.push_back(o);
  }
  Cloud ds;
  voxel_grid(raw, leaf, ds, true);
  for (const PointI &p : ds) {
    double C[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    if (with_ua) {
      const int idx = (int)p.intensity;
      const Pose pe = to_pose(ext7 + 7 * idx);
      eval_point_uncertainty_d(associate(p, pose_inv(pe)), pe, ext_cov36 + 36 * idx, cov_meas9, C);
      if (C[0][0] + C[1][1] + C[2][2] > trace_threshold) continue;
    }
    out.push_back(p);
    const float c6[6] = {(float)C[0][0], (float)C[0][1], (float)C[0][2], (float)C[1][1], (float)C[1][2], (float)C[2][2]};
    for (float v : c6) cov6.push_back(v);
  }
}

struct OutlierMapper {
  Mapper m;
  std::vector<Cloud> outlier;  // outlier_cloud_keyframes_cov (points; cloudUCTAssociateToMap reads the points only)
};

struct OutlierGlobalMap {
  std::vector<int> chosen;
  CovCloud map[2];
};

void append(CovCloud &dst, const CovCloud &src) {
  dst.pts.insert(dst.pts.end(), src.pts.begin(), src.pts.end());
  dst.cov6.insert(dst.cov6.end(), src.cov6.begin(), src.cov6.end());
  dst.trace.insert(dst.trace.end(), src.trace.begin(), src.trace.end());
}

// tests/host/orc_global_map.cpp's global_map with the outlier appends
void global_map(const OutlierMapper &om, int mode, const double *center7, double radius, float kf_leaf, float leaf, OutlierGlobalMap &g) {
  const Mapper &m = om.m;
  g = OutlierGlobalMap();
  if (m.kfs.empty()) return;  // :796
  Cloud sel, sel_ds;
  if (mode == 0) {
    const PointI q{(float)center7[0], (float)center7[1], (float)center7[2], 0.f};
    const float r2 = (float)(radius * radius);
    std::vector<std::pair<float, int>> found;
    for (const Keyframe &k : m.kfs) {
      float d2 = 0.f;
      const float a = k.pos.x - q.x, b = k.pos.y - q.y, c = k.pos.z - q.z;
      d2 += a * a, d2 += b * b, d2 += c * c;
      if (d2 < r2) found.push_back({d2, (int)k.pos.intensity});
    }
    std::sort(found.begin(), found.end());
    for (const auto &f : found) sel.push_back(m.kfs[f.second].pos);
  } else {
    for (const Keyframe &k : m.kfs) sel.push_back(k.pos);
  }
  voxel_grid(sel, kf_leaf, sel_ds, true);
  CovCloud raw[2];
  for (const PointI &p : sel_ds) {
    const int id = (int)p.intensity;
    g.chosen.push_back(id);
    CovCloud s, c, o;
    m.associate_kf(m.kfs[id], m.kfs[id].surf, s);
    m.associate_kf(m.kfs[id], m.kfs[id].corner, c);
    m.associate_kf(m.kfs[id], om.outlier[id], o);
    if (mode == 0) append(raw[0], s), append(raw[0], c), append(raw[0], o);  // :818-827
    else append(raw[0], s), append(raw[0], o), append(raw[1], c);            // :873-882
  }
  voxel_grid_cov(raw[0], leaf, (float)m.trace_thr, g.map[0]);
  if (mode == 1) voxel_grid_cov(raw[1], leaf, (float)m.trace_thr, g.map[1]);
}

}  // namespace

extern "C" {

// laser_cloud_outlier_cov of a rig frame (the inputs of orc_ua_frame_multi): out (capacity n_lidars points) and cov6, *n_out.
// ext_cov36 (n_lidars x 36) is read with with_ua only.
void orc_outlier_frame(const float *cloud, int n, const int *scan_start, int n_scans, int n_lidars, const double *ext7, const double *ext_cov36,
                       const double *cov_meas9, int with_ua, double trace_threshold, float leaf, float *out, float *out_cov6, int *n_out) {
  Cloud o;
  std::vector<float> c6;
  frame_outlier(cloud, n, scan_start, n_scans, n_lidars, ext7, ext_cov36, cov_meas9, with_ua != 0, trace_threshold, leaf, o, c6);
  *n_out = (int)o.size();
  if (!o.empty()) std::memcpy(out, o.data(), sizeof(PointI) * o.size()), std::memcpy(out_cov6, c6.data(), sizeof(float) * c6.size());
}

void *orc_outlier_mapper_create(double distance_keyframes, double orientation_keyframes_deg, double radius, double sur_kf_res,
                                double trace_threshold, float surf_leaf, float corner_leaf) {
  OutlierMapper *om = new OutlierMapper();
  Mapper *m = static_cast<Mapper *>(orc_mapper_create(distance_keyframes, orientation_keyframes_deg, radius, sur_kf_res, trace_threshold,
                                                      surf_leaf, corner_leaf));
  om->m = *m;
  orc_mapper_destroy(m);
  return om;
}
void orc_outlier_mapper_destroy(void *h) { delete static_cast<OutlierMapper *>(h); }
void orc_outlier_mapper_set_lidars(void *h, int n_lasers, const double *ext7, const double *ext_cov36, const double *cov_meas9, int with_ua) {
  orc_mapper_set_lidars(&static_cast<OutlierMapper *>(h)->m, n_lasers, ext7, ext_cov36, cov_meas9, with_ua);
}
// saveKeyframe with the three clouds (:641-683); margins2 as orc_mapper_save
int orc_outlier_mapper_save(void *h, const double *pose7, const double *cov36, const float *surf, int n_surf, const float *corner, int n_corner,
                            const float *outlier, int n_outlier, double *margins2) {
  OutlierMapper *om = static_cast<OutlierMapper *>(h);
  const int s = orc_mapper_save(&om->m, pose7, cov36, surf, n_surf, corner, n_corner, margins2);
  if (s) om->outlier.push_back(cloud_of(outlier, n_outlier));
  return s;
}
// as orc_global_map (counts[3]: chosen ids, map 0 size, map 1 size); returns a result handle
void *orc_outlier_global_map(void *h, int mode, const double *center7, double radius, double kf_leaf, float leaf, int *counts) {
  OutlierGlobalMap *g = new OutlierGlobalMap();
  global_map(*static_cast<const OutlierMapper *>(h), mode, center7, radius, (float)kf_leaf, leaf, *g);
  counts[0] = (int)g->chosen.size(), counts[1] = (int)g->map[0].pts.size(), counts[2] = (int)g->map[1].pts.size();
  return g;
}
void orc_outlier_global_map_read(void *r, int which, int *chosen, float *pts, float *cov6) {
  const OutlierGlobalMap *g = static_cast<const OutlierGlobalMap *>(r);
  const CovCloud &c = g->map[which];
  if (chosen) std::copy(g->chosen.begin(), g->chosen.end(), chosen);
  if (pts && !c.pts.empty()) std::memcpy(pts, c.pts.data(), sizeof(PointI) * c.pts.size());
  if (cov6 && !c.cov6.empty()) std::memcpy(cov6, c.cov6.data(), sizeof(float) * c.cov6.size());
}
void orc_outlier_global_map_free(void *r) { delete static_cast<OutlierGlobalMap *>(r); }

}  // extern "C"
