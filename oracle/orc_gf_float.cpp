// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// C entry points of liborc_gf_float.so (gf_float.mk): evalFullHessian for one feature set, and scan2MapOptimization with
// FLAGS_gf_method "gd_float" over consecutive frames, the mapper's state kept between the calls.  Clouds, poses and opts as in
// orc_capi.hpp.  Never linked into the product library.
#include "orc_gf_float.hpp"

using namespace orc;

namespace {
bool g_on = false;
float g_thre = 0.f;
GfFloatState g_state;

std::vector<double> traces(const float *cov6, int n) {  // extractCov: float cov_vec -> Matrix3d; trace in double
  std::vector<double> t(n);
  for (int i = 0; i < n; i++) t[i] = (double)cov6[i * 6] + (double)cov6[i * 6 + 3] + (double)cov6[i * 6 + 5];
  return t;
}
}  // namespace

extern "C" {

// H36 and *feat_num accumulate (in-out).  cov6 nullable (then default_trace), opts nullable (default match parameters).
void orc_full_hessian(int type, const float *map, int m, const float *scan, int n, const float *cov6, double default_trace,
                      const double *pose7, const double *opts, double *H36, int *feat_num) {
  Cloud mc = to_cloud(map, m), sc = to_cloud(scan, n);
  KdTree tree;
  tree.setInputCloud(&mc);
  std::vector<double> tr;
  if (cov6) tr = traces(cov6, n);
  eval_full_hessian((char)type, tree, mc, sc, to_pose(pose7), cov6 ? &tr : nullptr, default_trace, opts ? mp_from(opts) : MatchParams(), H36,
                    *feat_num);
}

// on = 1 starts the mapper's state (frame_cnt 0, gf_ratio_cur = min(1, gf_ratio_ini)), on = 0 ends the mode: orc_gf_float_scan2map is
// then orc_scan2map / orc_scan2map_ua (gd_fix)
void orc_gf_float_set(int on, float map_deg_thre, double gf_ratio_ini) {
  g_on = on != 0, g_thre = map_deg_thre;
  g_state = GfFloatState();
  g_state.ratio_cur = std::min(1.0, gf_ratio_ini);
}
// MAP_DEG_THRE alone, the state kept
void orc_gf_float_threshold(float map_deg_thre) { g_thre = map_deg_thre; }
// out5: frame_cnt, gf_ratio_cur, gf_deg_factor and total_feat_num of the last evaluation, whether the last frame evaluated
void orc_gf_float_get(double *out5) {
  out5[0] = (double)g_state.frame_cnt, out5[1] = g_state.ratio_cur, out5[2] = g_state.deg_factor, out5[3] = g_state.total_feat_num;
  out5[4] = g_state.evaluated;
}

// One mapper frame from its down-sampled scans on: scan2MapOptimization with opts' gf_method (3) and gf_ratio = FLAGS_gf_ratio_ini.
// surf_cov6 / corner_cov6 (both or neither): with_ua, per scan point cov_vec.  stats[16] as orc_scan2map; H36 nullable.
void orc_gf_float_scan2map(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_scan, int n_ss,
                           const float *surf_cov6, const float *corner_scan, int n_cs, const float *corner_cov6, const double *pose_init7,
                           const double *opts, double *pose_out7, double *stats, double *H36) {
  Scan2MapOptions o = opts_from(opts);
  std::vector<double> ts, tc;
  if (surf_cov6 && corner_cov6) {
    ts = traces(surf_cov6, n_ss), tc = traces(corner_cov6, n_cs);
    o.surf_cov_trace = &ts, o.corner_cov_trace = &tc;
  }
  Cloud sm = to_cloud(surf_map, n_sm), cm = to_cloud(corner_map, n_cm), ss = to_cloud(surf_scan, n_ss), cs = to_cloud(corner_scan, n_cs);
  const Pose init = to_pose(pose_init7);
  if (g_on) o = gf_float_begin(g_state, g_thre, sm, cm, ss, cs, init, o);
  Scan2MapResult r = scan2map(sm, cm, ss, cs, init, o);
  pose_to_param(r.pose, pose_out7);
  if (stats) {
    stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
    stats[5] = r.degenerate, stats[6] = r.t_kdtree, stats[7] = r.t_match, stats[8] = r.t_solver;
    for (int i = 0; i < 6; i++) stats[9 + i] = r.eig_last[i];
    stats[15] = 0;
  }
  if (H36) std::memcpy(H36, r.H_last, sizeof(r.H_last));
}

}  // extern "C"
