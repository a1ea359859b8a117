// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// FLAGS_gf_method "gd_float": ActiveFeatureSelection::evalFullHessian (estimator/src/lidarMapper/lidar_mapper.h:176-227) and the ratio
// policy around it in scan2MapOptimization (lidar_mapper_keyframe.cpp:456-495; frame_cnt++ :1059, initial ratio :1248).
//
// gd_float is gd_fix (orc_gf.hpp, GF_GD) called with a ratio that every 10th mapper frame re-decides.  The evaluation runs at
// iter_cnt == 0, before anything of the frame has moved pose_wmap_curr, and only sets gf_ratio_cur, which every goodFeatureMatching
// call of that frame then reads.  So a gd_float frame is: count the frame, evaluate at the initial pose if it is due and the map
// gate (:429) passes, then orc::scan2map with gf_ratio = gf_ratio_cur — the restatements of the steps stay the ones of orc_gf.hpp
// and orc_pipeline.hpp.
#pragma once
#include <algorithm>

#include "orc_capi.hpp"

namespace orc {

// evalFullHessian: every feature matched with n_neigh = 5, CHECK_FOV false (:187-211), the row of evaluateFeatJacobianMatching with the
// point's own covariance (:213-215); the caller's mat_H and feat_num accumulate J^T J and the count of the matched ones, feature by
// feature in index order (:216, :218).  Matching and rows are good_feature_matching's; its wo_gf selection is not used.
inline void eval_full_hessian(char type, const KdTree &tree, const Cloud &map, const Cloud &scan, const Pose &pose,
                              const std::vector<double> *cov_trace, double default_trace, const MatchParams &mp, double H[36], int &feat_num) {
  std::vector<Feature> all;
  std::vector<unsigned char> matched;
  std::vector<double> jaco;
  std::vector<int> sel;
  double sub_H[36];
  good_feature_matching(type, tree, map, scan, pose, cov_trace, default_trace, GF_WO, 1.0, 0, 5, mp, all, matched, jaco, sel, sub_H);
  for (size_t i = 0; i < scan.size(); i++) {
    if (!matched[i]) continue;
    gf_add_outer(H, jaco.data() + i * 6);  // mat_H = mat_H + jaco^T * jaco
    feat_num++;
  }
}

// what the mapper carries from frame to frame
struct GfFloatState {
  long long frame_cnt = 0;
  double ratio_cur = 1.0;    // gf_ratio_cur, min(1.0, FLAGS_gf_ratio_ini) at start (:1248)
  double deg_factor = 0.0;   // gf_deg_factor of the last evaluation (gf_deg_factor_list.back())
  int total_feat_num = 0;    // of the last evaluation
  int evaluated = 0;         // the last frame evaluated
};

// The part of a gd_float frame that precedes the Solve: frame_cnt++ (:1059, before the gate), and on every 10th frame that passes the
// map gate the evaluation — surf, then corner into one mat_H = 1e-6 I (:461-467) — and the decision (:470-492; MAP_DEG_THRE is a
// float, parameters.h:124; <= takes the 0.8 branch).  o.gf_ratio is FLAGS_gf_ratio_ini.  Returns o with gf_ratio = gf_ratio_cur.
inline Scan2MapOptions gf_float_begin(GfFloatState &g, float map_deg_thre, const Cloud &surf_map, const Cloud &corner_map, const Cloud &surf_scan,
                                      const Cloud &corner_scan, const Pose &pose_init, const Scan2MapOptions &o) {
  g.frame_cnt++;
  g.evaluated = 0;
  if ((surf_map.size() > 50) && (corner_map.size() > 10) && g.frame_cnt % 10 == 0) {
    KdTree kd_surf, kd_corner;
    kd_surf.setInputCloud(&surf_map);
    kd_corner.setInputCloud(&corner_map);
    double mat_H[36];
    for (int i = 0; i < 36; i++) mat_H[i] = (i % 7 == 0) ? 1e-6 : 0.0;
    g.total_feat_num = 0;
    if (o.point_plane) eval_full_hessian('s', kd_surf, surf_map, surf_scan, pose_init, o.surf_cov_trace, o.cov_trace, o.mp, mat_H, g.total_feat_num);
    if (o.point_edge) eval_full_hessian('c', kd_corner, corner_map, corner_scan, pose_init, o.corner_cov_trace, o.cov_trace, o.mp, mat_H, g.total_feat_num);
    g.deg_factor = logdet_chol(6, mat_H);
    g.ratio_cur = g.deg_factor > (double)map_deg_thre ? o.gf_ratio : 0.8;
    g.evaluated = 1;
  }
  Scan2MapOptions o2 = o;
  o2.gf_ratio = g.ratio_cur;
  return o2;
}

}  // namespace orc
