// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The global map of lidar_mapper_keyframe.cpp restated over the keyframe store (orc_mapper.hpp's Mapper):
//   pubGlobalMap   :780-851 (orc_global_map mode 0): radiusSearch(pose_point_cur, GLOBALMAP_KF_RADIUS) over
//                  pose_keyframes_3d (:804-808) -> down_size_filter_global_map_keyframes (:809-810) -> per chosen keyframe
//                  surf, corner, outlier through cloudUCTAssociateToMap, appended to one cloud (:814-828) ->
//                  down_size_filter_global_map_cov(MAP_SURF_RES, TRACE_THRESHOLD_MAPPING) (:840-843)
//   saveGlobalMap  :853-919 (mode 1): every keyframe (:862-863) -> the same position filter (:864-865) -> surf then outlier
//                  into the surf map, corner into the corner map (:866-882) -> both filtered at 2 * MAP_SURF_RES (:894-899)
// Restatement choices (in addition to orc_mapper.cpp's):
//   - the global map's radius search is extractSurroundingKeyFrames' (float d2 < (float)(radius^2), ascending (d2, id)) around the
//     caller's centre, the float PointI of a pose (pose_point_cur is the position saveKeyframe last tested, :643-645);
//   - down_size_filter_global_map_keyframes is VoxelGridCovarianceMLOAM<PointI> with leaf kf_leaf (10 m, :1293) over positions whose
//     intensity is the keyframe id: the last listed keyframe of a voxel gives the id;
//   - saveGlobalMap does not clear global_map_keyframes (:858-863): when the publisher thread has run, its last radius set sits in front
//     of the keyframe list.  Restated is the state in which it has not run: the list starts empty;
//   - a keyframe saved without an outlier cloud keeps an empty one, so its outlier appends add nothing.
#include "orc_mapper.hpp"

using namespace orc;

namespace {

struct GlobalMap {
  std::vector<int> chosen;
  CovCloud map[2];
};

// pubGlobalMap (mode 0, around center7) / saveGlobalMap (mode 1) of the store's keyframes
void global_map(const Mapper &m, int mode, const double *center7, double radius, float kf_leaf, float leaf, GlobalMap &g) {
  g = GlobalMap();
  if (m.kfs.empty()) return;  // :796
  Cloud sel, sel_ds;          // global_map_keyframes, global_map_keyframes_ds
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
    m.associate_kf(m.kfs[id], m.kfs[id].outlier, o);
    if (mode == 0) Mapper::append(raw[0], s), Mapper::append(raw[0], c), Mapper::append(raw[0], o);  // :818-827
    else Mapper::append(raw[0], s), Mapper::append(raw[0], o), Mapper::append(raw[1], c);            // :873-882
  }
  voxel_grid_cov(raw[0], leaf, (float)m.trace_thr, g.map[0]);
  if (mode == 1) voxel_grid_cov(raw[1], leaf, (float)m.trace_thr, g.map[1]);
}

}  // namespace

extern "C" {

// the global map of mapper h in mode 0 (pubGlobalMap, around center7) or 1 (saveGlobalMap); returns a result handle.
// counts[3]: chosen ids, map 0 size, map 1 size.
void *orc_global_map(void *h, int mode, const double *center7, double radius, double kf_leaf, float leaf, int *counts) {
  GlobalMap *g = new GlobalMap();
  global_map(*static_cast<const Mapper *>(h), mode, center7, radius, (float)kf_leaf, leaf, *g);
  counts[0] = (int)g->chosen.size(), counts[1] = (int)g->map[0].pts.size(), counts[2] = (int)g->map[1].pts.size();
  return g;
}
// chosen ids (nullable) and map `which` (points and cov_vec, nullable), sized by orc_global_map's counts
void orc_global_map_read(void *r, int which, int *chosen, float *pts, float *cov6) {
  const GlobalMap *g = static_cast<const GlobalMap *>(r);
  const CovCloud &c = g->map[which];
  if (chosen) std::copy(g->chosen.begin(), g->chosen.end(), chosen);
  if (pts && !c.pts.empty()) std::memcpy(pts, c.pts.data(), sizeof(PointI) * c.pts.size());
  if (cov6 && !c.cov6.empty()) std::memcpy(cov6, c.cov6.data(), sizeof(float) * c.cov6.size());
}
void orc_global_map_free(void *r) { delete static_cast<GlobalMap *>(r); }

}  // extern "C"
