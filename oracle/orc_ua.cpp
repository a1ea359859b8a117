// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The uncertainty-aware mapper (with_ua = true) of lidar_mapper_keyframe.cpp as flat C entry points for tests/uncertainty_lib.py,
// built next to liborc.so from the same headers (liborc_ua.so):
//   downsampleCurrentScan's uncertainty loop (:356-421): per down-sampled point idx = int(intensity), pointAssociateToMap with
//     pose_ext[idx]^-1, evalPointUncertainty under pose_ext[idx] (associate_uct.hpp:196-215), dropped when the double trace >
//     TRACE_THRESHOLD_MAPPING, kept in order with the float cov;
//   sqrt_info of every residual from its point's covariance (extractCov + clamp, :541-560, lidar_map_factor.hpp:34,41);
//   cov_mapping = mat_H.inverse() after the last Solve (:600-610): H = problem.Evaluate at the returned pose with the residual blocks
//     of the last association.
// Restatement choices (in addition to orc_math.hpp's):
//   - the 6x6 inverse is an unblocked partial-pivot LU (first largest |pivot| of the column, row swap, multipliers divided by the
//     pivot, rank-1 update of the trailing block) solved column by column — Eigen's algorithm, not its blocked kernels;
//   - when the last evaluation has no residual rows the covariance is zero, where Eigen would return inf / NaN;
//   - the last association is recovered by re-running orc::scan2map with one GN iteration fewer (deterministic) and matching at its
//     pose, so the restatement of the Solve itself stays the one of orc_pipeline.hpp.
#include "orc_pipeline.hpp"
#include "orc_gf.hpp"
#include "orc_uct.hpp"

using namespace orc;

namespace {

Cloud to_cloud(const float *p, int n) {
  Cloud c(n);
  if (n > 0) std::memcpy(c.data(), p, sizeof(PointI) * (size_t)n);
  return c;
}
Pose to_pose(const double *x) { return Pose{Q4{x[3], x[4], x[5], x[6]}, V3{x[0], x[1], x[2]}}; }

// opts layout of orc_capi.cpp (orc_default_opts)
enum {
  O_MAX_OUTER = 0, O_MAX_INNER, O_HUBER, O_EIG_THRE, O_N_NEIGH, O_CHECK_FOV, O_POINT_PLANE, O_POINT_EDGE,
  O_COV_TRACE, O_DIST_SQ_THR, O_NEARBY_SCAN, O_MIN_MATCH_SQ, O_MIN_PLANE_DIS, O_GF_METHOD, O_GF_RATIO, O_GF_SEED, O_COUNT
};
Scan2MapOptions opts_from(const double *opts) {
  Scan2MapOptions o;
  o.max_outer = (int)opts[O_MAX_OUTER], o.max_inner = (int)opts[O_MAX_INNER], o.huber_a = opts[O_HUBER];
  o.eig_thre = opts[O_EIG_THRE], o.n_neigh = (int)opts[O_N_NEIGH], o.check_fov = opts[O_CHECK_FOV] != 0;
  o.point_plane = opts[O_POINT_PLANE] != 0, o.point_edge = opts[O_POINT_EDGE] != 0, o.cov_trace = opts[O_COV_TRACE];
  o.mp.distance_sq_threshold = (float)opts[O_DIST_SQ_THR], o.mp.nearby_scan = (float)opts[O_NEARBY_SCAN];
  o.mp.min_match_sq_dis = (float)opts[O_MIN_MATCH_SQ], o.mp.min_plane_dis = (float)opts[O_MIN_PLANE_DIS];
  o.gf_method = (int)opts[O_GF_METHOD], o.gf_ratio = opts[O_GF_RATIO], o.gf_seed = (uint64_t)opts[O_GF_SEED];
  return o;
}

void lu_inverse6(const double *H, double *out) {
  double A[36];
  int perm[6];
  for (int i = 0; i < 36; i++) A[i] = H[i];
  for (int i = 0; i < 6; i++) perm[i] = i;
  for (int k = 0; k < 6; k++) {
    int piv = k;
    double best = std::fabs(A[k * 6 + k]);
    for (int i = k + 1; i < 6; i++)
      if (std::fabs(A[i * 6 + k]) > best) best = std::fabs(A[i * 6 + k]), piv = i;
    if (piv != k) {
      for (int j = 0; j < 6; j++) std::swap(A[k * 6 + j], A[piv * 6 + j]);
      std::swap(perm[k], perm[piv]);
    }
    if (A[k * 6 + k] != 0.0)
      for (int i = k + 1; i < 6; i++) A[i * 6 + k] /= A[k * 6 + k];
    for (int i = k + 1; i < 6; i++)
      for (int j = k + 1; j < 6; j++) A[i * 6 + j] -= A[i * 6 + k] * A[k * 6 + j];
  }
  for (int col = 0; col < 6; col++) {
    double y[6];
    for (int i = 0; i < 6; i++) {  // L y = P e_col (unit lower)
      double s = perm[i] == col ? 1.0 : 0.0;
      for (int j = 0; j < i; j++) s -= A[i * 6 + j] * y[j];
      y[i] = s;
    }
    for (int i = 5; i >= 0; i--) {  // U x = y
      double s = y[i];
      for (int j = i + 1; j < 6; j++) s -= A[i * 6 + j] * y[j];
      y[i] = s / A[i * 6 + i];
    }
    for (int i = 0; i < 6; i++) out[i * 6 + col] = y[i];
  }
}

// scan2MapOptimization with with_ua = true (o.surf_cov_trace / o.corner_cov_trace set): the Solve of orc::scan2map, then
// cov_mapping = H^-1 with H evaluated at the returned pose over the residual blocks of the last association (:600-610).
Scan2MapResult scan2map_with_cov(const Cloud &sm, const Cloud &cm, const Cloud &ss, const Cloud &cs, const Pose &init, const Scan2MapOptions &o,
                                 double cov[36], double H[36]) {
  std::memset(cov, 0, 36 * sizeof(double));
  std::memset(H, 0, 36 * sizeof(double));
  Scan2MapResult r = scan2map(sm, cm, ss, cs, init, o);
  if (!r.ran || o.max_outer < 1) return r;  // map gate (:637): zero
  Pose assoc = init;  // pose_wmap_curr at the start of the last GN iteration
  if (o.max_outer > 1) {
    Scan2MapOptions o2 = o;
    o2.max_outer = o.max_outer - 1;
    assoc = scan2map(sm, cm, ss, cs, init, o2).pose;
  }
  KdTree kd_surf, kd_corner;
  kd_surf.setInputCloud(&sm);
  kd_corner.setInputCloud(&cm);
  std::vector<Feature> corner_f, surf_f;
  const uint64_t it = (uint64_t)(o.max_outer - 1);
  if (o.gf_method == 0) {
    if (o.point_edge) match_from_map('c', kd_corner, cm, cs, assoc, corner_f, o.n_neigh, o.check_fov, o.mp);
    if (o.point_plane) match_from_map('s', kd_surf, sm, ss, assoc, surf_f, o.n_neigh, o.check_fov, o.mp);
  } else {
    std::vector<Feature> all;
    std::vector<unsigned char> mt;
    std::vector<double> jc;
    std::vector<int> sel;
    double subH[36];
    if (o.point_edge) {
      good_feature_matching('c', kd_corner, cm, cs, assoc, o.corner_cov_trace, o.cov_trace, o.gf_method, o.gf_ratio, o.gf_seed + 2 * it, o.n_neigh,
                            o.mp, all, mt, jc, sel, subH);
      for (int q : sel) corner_f.push_back(all[q]);
    }
    if (o.point_plane) {
      good_feature_matching('s', kd_surf, sm, ss, assoc, o.surf_cov_trace, o.cov_trace, o.gf_method, o.gf_ratio, o.gf_seed + 2 * it + 1, o.n_neigh,
                            o.mp, all, mt, jc, sel, subH);
      for (int q : sel) surf_f.push_back(all[q]);
    }
  }
  double para[7];
  pose_to_param(r.pose, para);
  Problem problem;
  problem.huber_a = o.huber_a;
  const int pid = problem.add_param(para);
  const double sinfo = map_sqrt_info(o.cov_trace);
  for (const Feature &f : surf_f) {  // the order of orc::scan2map (:537-549, then :552-571)
    const double si = o.surf_cov_trace ? map_sqrt_info((*o.surf_cov_trace)[f.idx]) : sinfo;
    problem.blocks.push_back(ResidualBlock{F_PLANE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], 0, 0}, si, {pid, 0, 0}});
  }
  for (const Feature &f : corner_f) {
    const double si = o.corner_cov_trace ? map_sqrt_info((*o.corner_cov_trace)[f.idx]) : sinfo;
    problem.blocks.push_back(
        ResidualBlock{F_EDGE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], f.coeffs[4], f.coeffs[5]}, si, {pid, 0, 0}});
  }
  NormalEq ne;
  std::vector<const double *> xs{para};
  problem.evaluate(xs, true, ne);
  if (ne.rows > 0) {
    std::memcpy(H, ne.H.data(), 36 * sizeof(double));
    lu_inverse6(H, cov);
  }
  return r;
}

// transformCloudFeature + merge + downsampleCurrentScan of a multi-LiDAR frame, as orc_capi.cpp's prepare_multi
void prepare_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                   float corner_leaf, float surf_leaf, Cloud &cs, Cloud &ss) {
  const int R = n_scans / n_lidars;
  std::vector<CloudFeature> feats(n_lidars);
  for (int l = 0; l < n_lidars; l++) {
    const int lo = scan_start[l * R] - 5, hi = (l + 1 < n_lidars) ? scan_start[(l + 1) * R] - 5 : n;
    Cloud c = to_cloud(cloud + 4 * (size_t)lo, hi - lo);
    ScanInfo si;
    for (int r = 0; r < R; r++) si.scan_start_ind.push_back(scan_start[l * R + r] - lo), si.scan_end_ind.push_back(scan_end[l * R + r] - lo);
    extract_cloud(c, si, R, feats[l]);
  }
  Cloud corner, surf;
  for (int l = 0; l < n_lidars; l++) {
    const double *e = ext7 + 7 * l;
    const Pose T = make_pose(Q4{e[3], e[4], e[5], e[6]}, V3{e[0], e[1], e[2]});
    const M3 Rm = qmat(T.q);
    float m[12];
    for (int r = 0; r < 3; r++) {
      for (int k = 0; k < 3; k++) m[4 * r + k] = (float)Rm(r, k);
      m[4 * r + 3] = (float)(r == 0 ? T.t.x : (r == 1 ? T.t.y : T.t.z));
    }
    auto xf = [&](const Cloud &in, Cloud &out) {
      for (const PointI &p : in) {
        PointI o;
        o.x = m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3];
        o.y = m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7];
        o.z = m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11];
        o.intensity = (float)l;
        out.push_back(o);
      }
    };
    xf(feats[l].corner_points_less_sharp, corner);
    xf(feats[l].surf_points_less_flat, surf);
  }
  voxel_grid(corner, corner_leaf, cs, true);
  voxel_grid(surf, surf_leaf, ss, true);
}

}  // namespace

extern "C" {

// ---- the multi-LiDAR frame with with_ua = true.  ext_cov36: n_lidars x 36 (pose_ext[l].cov_, [translation | rotation]).
// stats[20] as orc_frame_multi ([18], [19]: gated counts; timings 0); cov36: cov_mapping; H36 (nullable): the H it inverts;
// the gated scans (capacity n each, nullable) with their cov_vec.
void orc_ua_frame_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                        const double *ext_cov36, const double *cov_meas9, double trace_threshold, const float *surf_map, int n_sm,
                        const float *corner_map, int n_cm, float corner_leaf, float surf_leaf, const double *pose_init7, const double *opts,
                        double *pose_out7, double *stats, double *cov36, double *H36, float *surf_out, float *surf_cov6, int *n_surf,
                        float *corner_out, float *corner_cov6, int *n_corner) {
  Cloud cs, ss;
  prepare_multi(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, corner_leaf, surf_leaf, cs, ss);
  auto gate = [&](const Cloud &in, Cloud &out, std::vector<float> &cov6, std::vector<double> &tr) {
    for (const PointI &p : in) {
      const int idx = (int)p.intensity;
      const Pose pe = to_pose(ext7 + 7 * idx);
      const PointI sel = associate(p, pose_inv(pe));
      double C[3][3];
      eval_point_uncertainty_d(sel, pe, ext_cov36 + 36 * idx, cov_meas9, C);
      if (C[0][0] + C[1][1] + C[2][2] > trace_threshold) continue;
      out.push_back(p);
      const float c6[6] = {(float)C[0][0], (float)C[0][1], (float)C[0][2], (float)C[1][1], (float)C[1][2], (float)C[2][2]};
      for (float v : c6) cov6.push_back(v);
      tr.push_back((double)c6[0] + (double)c6[3] + (double)c6[5]);  // extractCov: float cov_vec -> Matrix3d, trace in double
    }
  };
  Cloud sg, cg;
  std::vector<float> sc6, cc6;
  std::vector<double> st, ct;
  gate(ss, sg, sc6, st);
  gate(cs, cg, cc6, ct);
  Scan2MapOptions o = opts_from(opts);
  o.surf_cov_trace = &st, o.corner_cov_trace = &ct;
  double cov[36], H[36];
  Scan2MapResult r = scan2map_with_cov(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), sg, cg, to_pose(pose_init7), o, cov, H);
  pose_to_param(r.pose, pose_out7);
  if (stats) {
    for (int i = 0; i < 20; i++) stats[i] = 0;
    stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
    stats[5] = r.degenerate;
    for (int i = 0; i < 6; i++) stats[9 + i] = r.eig_last[i];
    stats[18] = (double)sg.size(), stats[19] = (double)cg.size();
  }
  if (cov36) std::memcpy(cov36, cov, sizeof(cov));
  if (H36) std::memcpy(H36, H, sizeof(H));
  if (n_surf) *n_surf = (int)sg.size();
  if (n_corner) *n_corner = (int)cg.size();
  if (surf_out && !sg.empty()) std::memcpy(surf_out, sg.data(), sizeof(PointI) * sg.size());
  if (surf_cov6 && !sc6.empty()) std::memcpy(surf_cov6, sc6.data(), sizeof(float) * sc6.size());
  if (corner_out && !cg.empty()) std::memcpy(corner_out, cg.data(), sizeof(PointI) * cg.size());
  if (corner_cov6 && !cc6.empty()) std::memcpy(corner_cov6, cc6.data(), sizeof(float) * cc6.size());
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
