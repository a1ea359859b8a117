// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The pieces the C entry points of liborc.so share (orc_capi.cpp, orc_ua.cpp, orc_mapper.cpp, orc_global_map.cpp):
//   - the C-API marshalling: float32 [n,4] clouds, double[7] [tx ty tz qx qy qz qw] poses, the opts layout (orc_default_opts);
//   - the float rig transform of transformCloudFeature (visualization.cpp:40-52);
//   - TransformToEnd (utility.h:54-100), the undistortion of the odometry's DISTORTION step;
//   - the rig's feature prepare step (estimator.cpp:249-263 -> pubPointCloud -> downsampleCurrentScan's filters);
//   - downsampleCurrentScan's with_ua gate (lidar_mapper_keyframe.cpp:356-421);
//   - the mapper-side frame (frame_ua) with its with_ua Solve and cov_mapping (scan2map_with_cov; restatement choices in orc_ua.cpp).
#pragma once
#include "orc_pipeline.hpp"
#include "orc_gf.hpp"
#include "orc_uct.hpp"
#include <cfloat>

namespace orc {

inline Cloud to_cloud(const float *p, int n) {
  Cloud c(n);
  if (n > 0) std::memcpy(c.data(), p, sizeof(PointI) * (size_t)n);
  return c;
}
inline Pose to_pose(const double *x) { return Pose{Q4{x[3], x[4], x[5], x[6]}, V3{x[0], x[1], x[2]}}; }

// opts layout shared by the pipeline calls
enum {
  O_MAX_OUTER = 0, O_MAX_INNER, O_HUBER, O_EIG_THRE, O_N_NEIGH, O_CHECK_FOV, O_POINT_PLANE, O_POINT_EDGE,
  O_COV_TRACE, O_DIST_SQ_THR, O_NEARBY_SCAN, O_MIN_MATCH_SQ, O_MIN_PLANE_DIS, O_GF_METHOD, O_GF_RATIO, O_GF_SEED, O_COUNT
};
inline MatchParams mp_from(const double *o) {
  MatchParams mp;
  mp.distance_sq_threshold = (float)o[O_DIST_SQ_THR];
  mp.nearby_scan = (float)o[O_NEARBY_SCAN];
  mp.min_match_sq_dis = (float)o[O_MIN_MATCH_SQ];
  mp.min_plane_dis = (float)o[O_MIN_PLANE_DIS];
  return mp;
}
inline Scan2MapOptions opts_from(const double *opts) {
  Scan2MapOptions o;
  o.max_outer = (int)opts[O_MAX_OUTER], o.max_inner = (int)opts[O_MAX_INNER], o.huber_a = opts[O_HUBER];
  o.eig_thre = opts[O_EIG_THRE], o.n_neigh = (int)opts[O_N_NEIGH], o.check_fov = opts[O_CHECK_FOV] != 0;
  o.point_plane = opts[O_POINT_PLANE] != 0, o.point_edge = opts[O_POINT_EDGE] != 0, o.cov_trace = opts[O_COV_TRACE];
  o.mp = mp_from(opts);
  o.gf_method = (int)opts[O_GF_METHOD], o.gf_ratio = opts[O_GF_RATIO], o.gf_seed = (uint64_t)opts[O_GF_SEED];
  return o;
}

// pcl::transformPointCloud with Pose(q, t).T_.cast<float>() (Pose(q, t) normalises q, pose.cpp:34-41): PCL 1.8 transforms.hpp evaluates
// x' = m00 x + m01 y + m02 z + m03 in float.
struct FloatTransform {
  float m[12];
  explicit FloatTransform(const double *e7) {
    const Pose T = make_pose(Q4{e7[3], e7[4], e7[5], e7[6]}, V3{e7[0], e7[1], e7[2]});
    const M3 Rm = qmat(T.q);
    for (int r = 0; r < 3; r++) {
      for (int k = 0; k < 3; k++) m[4 * r + k] = (float)Rm(r, k);
      m[4 * r + 3] = (float)(r == 0 ? T.t.x : (r == 1 ? T.t.y : T.t.z));
    }
  }
  PointI operator()(const PointI &p, float intensity) const {
    PointI o;
    o.x = m[0] * p.x + m[1] * p.y + m[2] * p.z + m[3];
    o.y = m[4] * p.x + m[5] * p.y + m[6] * p.z + m[7];
    o.z = m[8] * p.x + m[9] * p.y + m[10] * p.z + m[11];
    o.intensity = intensity;
    return o;
  }
};

// TransformToEnd(p, p, pose, true, scan_period), pose as given (a Pose holds a normalised q).  Eigen 3.3's slerp (Identity.slerp(s, q):
// d = q.w, acos / sin of the C library, weights 1 - s and s when |d| >= 1 - DBL_EPSILON, the second weight negated when d < 0, the
// coefficients scale0 (0,0,0,1) + scale1 q NOT renormalised), _transformVector, Quaternion::inverse = conj / squaredNorm (summed x, y, z, w
// in order).  s = (float)(intensity - (float)int(intensity)) / (float)scan_period, the float expression of utility.h:64, widened to double.
inline PointI transform_point_to_end(const PointI &p, const Pose &pose, float scan_period) {
  const float fr = p.intensity - (float)(int)p.intensity;
  const double s = (double)(fr / scan_period);
  const Q4 &q = pose.q;
  const double d = q.w, absD = std::fabs(d), one = 1.0 - DBL_EPSILON;
  double s0, s1;
  if (absD >= one) {
    s0 = 1.0 - s, s1 = s;
  } else {
    const double theta = std::acos(absD), st = std::sin(theta);
    s0 = std::sin((1.0 - s) * theta) / st;
    s1 = std::sin(s * theta) / st;
  }
  if (d < 0.0) s1 = -s1;
  const Q4 qs{s0 * 0.0 + s1 * q.x, s0 * 0.0 + s1 * q.y, s0 * 0.0 + s1 * q.z, s0 * 1.0 + s1 * q.w};
  const V3 ts{s * pose.t.x, s * pose.t.y, s * pose.t.z};
  const V3 un = qrot(qs, V3{(double)p.x, (double)p.y, (double)p.z}) + ts;
  PointI tmp{(float)un.x, (float)un.y, (float)un.z, p.intensity};
  const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  const Q4 qi = n2 > 0.0 ? Q4{-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2} : Q4{0, 0, 0, 0};
  const V3 e = qrot(qi, V3{(double)tmp.x - pose.t.x, (double)tmp.y - pose.t.y, (double)tmp.z - pose.t.z});
  return PointI{(float)e.x, (float)e.y, (float)e.z, p.intensity};
}

inline void undistort_cloud(Cloud &c, const double *pose7, float scan_period) {
  const Pose p = to_pose(pose7);
  for (PointI &q : c) q = transform_point_to_end(q, p, scan_period);
}

// The features of a multi-LiDAR frame as they enter scan2MapOptimization: the concatenated sweeps of n_lidars LiDARs (LiDAR-major,
// n_scans = n_lidars x rings; scan_start / scan_end index the concatenation).  Per LiDAR l (estimator.cpp:249-263, OpenMP over the
// LiDARs): extractCloud on its rings; with poses7 (nullable, n_lidars x 7) undistortMeasurements (estimator.cpp:376-408) moves its
// corner_points_less_sharp and surf_points_less_flat with poses7[l]; transformCloudFeature with ext7[l] and intensity = l; `+=` LiDAR by
// LiDAR (pubPointCloud :93-104, ESTIMATE_EXTRINSIC == 0); then downsampleCurrentScan's two filters on the merged clouds.
// The per-LiDAR extraction is independent, so the result does not depend on the thread count.
inline void prepare_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                          const double *poses7, float scan_period, float corner_leaf, float surf_leaf, Cloud &cs, Cloud &ss, double *t_extract,
                          double *t_down) {
  const int R = n_scans / n_lidars;
  std::vector<CloudFeature> feats(n_lidars);
  double t0 = now_s();
#pragma omp parallel for schedule(dynamic, 1)
  for (int l = 0; l < n_lidars; l++) {
    // the LiDAR's own cloud: points [first ring begin - 5, last ring end + 6) of the concatenation (ScanInfo = ring_begin + 5 / ring_end - 6)
    const int lo = scan_start[l * R] - 5, hi = (l + 1 < n_lidars) ? scan_start[(l + 1) * R] - 5 : n;
    Cloud c = to_cloud(cloud + 4 * (size_t)lo, hi - lo);
    ScanInfo si;
    for (int r = 0; r < R; r++) si.scan_start_ind.push_back(scan_start[l * R + r] - lo), si.scan_end_ind.push_back(scan_end[l * R + r] - lo);
    extract_cloud(c, si, R, feats[l]);
  }
  Cloud corner, surf;
  for (int l = 0; l < n_lidars; l++) {
    if (poses7) {
      undistort_cloud(feats[l].corner_points_less_sharp, poses7 + 7 * l, scan_period);
      undistort_cloud(feats[l].surf_points_less_flat, poses7 + 7 * l, scan_period);
    }
    const FloatTransform xf(ext7 + 7 * l);
    for (const PointI &p : feats[l].corner_points_less_sharp) corner.push_back(xf(p, (float)l));
    for (const PointI &p : feats[l].surf_points_less_flat) surf.push_back(xf(p, (float)l));
  }
  double t1 = now_s();
  voxel_grid(corner, corner_leaf, cs, true);  // lidar_mapper_keyframe.cpp:359-364
  voxel_grid(surf, surf_leaf, ss, true);
  double t2 = now_s();
  if (t_extract) *t_extract = t1 - t0;
  if (t_down) *t_down = t2 - t1;
}

// downsampleCurrentScan's uncertainty loop (lidar_mapper_keyframe.cpp:356-421) over a down-sampled scan: per point idx = int(intensity),
// pointAssociateToMap with pose_ext[idx]^-1, evalPointUncertainty under pose_ext[idx] (associate_uct.hpp:196-215), dropped when the double
// trace > trace_threshold, kept in order with the float cov_vec.  ext_cov36 == nullptr (with_ua false): every point kept, cov_vec zero.
// trace (nullable): extractCov's trace of each kept cov_vec (float cov_vec -> Matrix3d, trace in double).
inline void ua_gate(const Cloud &in, const double *ext7, const double *ext_cov36, const double *cov_meas9, double trace_threshold, Cloud &out,
                    std::vector<float> &cov6, std::vector<double> *trace) {
  for (const PointI &p : in) {
    double C[3][3] = {{0, 0, 0}, {0, 0, 0}, {0, 0, 0}};
    if (ext_cov36) {
      const int idx = (int)p.intensity;
      const Pose pe = to_pose(ext7 + 7 * idx);
      eval_point_uncertainty_d(associate(p, pose_inv(pe)), pe, ext_cov36 + 36 * idx, cov_meas9, C);
      if (C[0][0] + C[1][1] + C[2][2] > trace_threshold) continue;
    }
    out.push_back(p);
    const float c6[6] = {(float)C[0][0], (float)C[0][1], (float)C[0][2], (float)C[1][1], (float)C[1][2], (float)C[2][2]};
    for (float v : c6) cov6.push_back(v);
    if (trace) trace->push_back((double)c6[0] + (double)c6[3] + (double)c6[5]);
  }
}

// the 6x6 inverse of cov_mapping (see orc_ua.cpp)
inline void lu_inverse6(const double *H, double *out) {
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
inline Scan2MapResult scan2map_with_cov(const Cloud &sm, const Cloud &cm, const Cloud &ss, const Cloud &cs, const Pose &init, const Scan2MapOptions &o,
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

// The features of one LiDAR's whole sweep entering downsampleCurrentScan's filters, without the rig merge: extractCloud, the undistortion
// with poses7 (nullable), pointAssociateToMap with single_ext7 (nullable), the two filters.
inline void prepare_single(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, const double *single_ext7,
                           const double *poses7, float scan_period, float corner_leaf, float surf_leaf, Cloud &cs, Cloud &ss) {
  CloudFeature f;
  ScanInfo si;
  si.scan_start_ind.assign(scan_start, scan_start + n_scans), si.scan_end_ind.assign(scan_end, scan_end + n_scans);
  extract_cloud(to_cloud(cloud, n), si, n_scans, f);
  Cloud corner = f.corner_points_less_sharp, surf = f.surf_points_less_flat;
  if (poses7) undistort_cloud(corner, poses7, scan_period), undistort_cloud(surf, poses7, scan_period);
  if (single_ext7) {
    const Pose T = to_pose(single_ext7);
    for (PointI &p : corner) p = associate(p, T);
    for (PointI &p : surf) p = associate(p, T);
  }
  voxel_grid(corner, corner_leaf, cs, true);
  voxel_grid(surf, surf_leaf, ss, true);
}

// The mapper-side frame (orc_frame_ua, orc_mapper_process): the features, the with_ua gate, the Solve.  ext7 (n_lidars x 7): the rig
// merge (prepare_multi); nullptr: the whole sweep is one LiDAR's, moved with single_ext7 (nullable).  poses7 (nullable): the undistortion, one pose per LiDAR.  ext_cov36 (n_lidars x 36, pose_ext[l].cov_,
// [translation | rotation]; nullable): with_ua, ext7 required.  stats[20] as orc_frame_multi ([18], [19]: gated counts; timings 0);
// cov36: cov_mapping (zero without with_ua); H36 (nullable): the H it inverts; the scans entering the solve (capacity n each, nullable)
// with their cov_vec.
inline void frame_ua(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                     const double *single_ext7, const double *poses7, float scan_period, const double *ext_cov36, const double *cov_meas9,
                     double trace_threshold, const float *surf_map, int n_sm, const float *corner_map, int n_cm, float corner_leaf,
                     float surf_leaf, const double *pose_init7, const double *opts, double *pose_out7, double *stats, double *cov36,
                     double *H36, float *surf_out, float *surf_cov6, int *n_surf, float *corner_out, float *corner_cov6, int *n_corner) {
  Cloud cs, ss;
  if (ext7)
    prepare_multi(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, poses7, scan_period, corner_leaf, surf_leaf, cs, ss, nullptr, nullptr);
  else
    prepare_single(cloud, n, scan_start, scan_end, n_scans, single_ext7, poses7, scan_period, corner_leaf, surf_leaf, cs, ss);
  Cloud sg, cg;
  std::vector<float> sc6, cc6;
  std::vector<double> st, ct;
  ua_gate(ss, ext7, ext_cov36, cov_meas9, trace_threshold, sg, sc6, &st);
  ua_gate(cs, ext7, ext_cov36, cov_meas9, trace_threshold, cg, cc6, &ct);
  Scan2MapOptions o = opts_from(opts);
  double cov[36] = {0}, H[36] = {0};
  Scan2MapResult r;
  if (ext_cov36) {
    o.surf_cov_trace = &st, o.corner_cov_trace = &ct;
    r = scan2map_with_cov(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), sg, cg, to_pose(pose_init7), o, cov, H);
  } else {
    r = scan2map(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), sg, cg, to_pose(pose_init7), o);
  }
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

}  // namespace orc
