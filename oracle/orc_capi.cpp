// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// Flat C entry points over the restatement so tests/ and bench.py's cpu_baseline leg can drive it
// through ctypes: the single steps, scan2MapOptimization, the whole frame (orc_frame / orc_frame_multi), the
// calibration step, the odometry solve and the tracker.  Clouds are float32 [n,4] (x,y,z,intensity); poses are
// double[7] [tx ty tz qx qy qz qw] (orc_capi.hpp).  Never linked into the product library.
#include "orc_capi.hpp"
#include "orc_segment.hpp"
#include <cstdio>
#include <dlfcn.h>
#ifdef _OPENMP
#include <omp.h>
#endif

using namespace orc;

std::vector<int> g_gf_groups_surf, g_gf_groups_corner;  // see orc_set_gf_groups

extern "C" {

// Timed CPU arm only: route KdTree through the reference's nanoflann (oracle/_ref/libref_knn.so).  path == null / ""
// switches back to the restatement's own tree.  Returns 1 when the backend is active.
int orc_use_ref_tree(const char *so_path) {
  RefTreeApi &api = ref_tree_api();
  api = RefTreeApi();
  if (!so_path || !so_path[0]) return 0;
  void *h = dlopen(so_path, RTLD_NOW | RTLD_LOCAL);
  if (!h) return 0;
  api.create = reinterpret_cast<void *(*)(const float *, int)>(dlsym(h, "ref_tree_create"));
  api.knn = reinterpret_cast<int (*)(void *, float, float, float, int, int *, float *)>(dlsym(h, "ref_tree_knn"));
  api.destroy = reinterpret_cast<void (*)(void *)>(dlsym(h, "ref_tree_destroy"));
  if (!api.create || !api.knn || !api.destroy) {
    api = RefTreeApi();
    return 0;
  }
  return 1;
}

int orc_num_opts() { return O_COUNT; }
void orc_default_opts(double *o) {
  Scan2MapOptions d;
  o[O_MAX_OUTER] = d.max_outer, o[O_MAX_INNER] = d.max_inner, o[O_HUBER] = d.huber_a, o[O_EIG_THRE] = d.eig_thre;
  o[O_N_NEIGH] = d.n_neigh, o[O_CHECK_FOV] = d.check_fov, o[O_POINT_PLANE] = d.point_plane, o[O_POINT_EDGE] = d.point_edge;
  o[O_COV_TRACE] = d.cov_trace, o[O_DIST_SQ_THR] = d.mp.distance_sq_threshold, o[O_NEARBY_SCAN] = d.mp.nearby_scan;
  o[O_MIN_MATCH_SQ] = d.mp.min_match_sq_dis, o[O_MIN_PLANE_DIS] = d.mp.min_plane_dis;
  o[O_GF_METHOD] = d.gf_method, o[O_GF_RATIO] = d.gf_ratio, o[O_GF_SEED] = (double)d.gf_seed;
}

// ---- small dense kernels (known-answer tests)
void orc_eig3f(const float *A9, float *w3, float *V9) { eig3f(A9, w3, V9); }
int orc_lsq_plane(const float *A, int K, float *n3) { return lsq_plane_f(A, K, n3) ? 1 : 0; }
void orc_eig_sym(int N, const double *A, double *w, double *V) { eig_sym(N, A, w, V); }
double orc_logdet(int N, const double *H) { return logdet_chol(N, H); }
void orc_huber(double a, double s, double *out2) { huber(a, s, &out2[0], &out2[1]); }
double orc_map_sqrt_info(double cov_trace) { return map_sqrt_info(cov_trace); }
void orc_associate(const float *pts, int n, const double *pose7, float *out) {
  Pose p = to_pose(pose7);
  for (int i = 0; i < n; i++) {
    PointI o = associate(PointI{pts[i * 4], pts[i * 4 + 1], pts[i * 4 + 2], pts[i * 4 + 3]}, p);
    out[i * 4] = o.x, out[i * 4 + 1] = o.y, out[i * 4 + 2] = o.z, out[i * 4 + 3] = o.intensity;
  }
}
void orc_pose_mul(const double *a7, const double *b7, double *out7) { pose_to_param(pose_mul(to_pose(a7), to_pose(b7)), out7); }
void orc_pose_inv(const double *a7, double *out7) { pose_to_param(pose_inv(to_pose(a7)), out7); }

// PoseLocalParameterization::Plus with optional V_update (row-major 6x6; null = identity)
void orc_plus(const double *x7, const double *delta6, const double *V36, double *out7) {
  PoseLocalParameterization lp;
  if (V36) std::memcpy(lp.V_update, V36, sizeof(lp.V_update));
  lp.Plus(x7, delta6, out7);
}
void orc_eval_degeneracy(const double *H36, double thre, double *V36, double *eig6, int *degenerate) {
  PoseLocalParameterization lp;
  eval_degeneracy(H36, thre, lp, eig6);
  std::memcpy(V36, lp.V_update, sizeof(lp.V_update));
  *degenerate = lp.is_degenerate ? 1 : 0;
}

// ---- kNN.  Missing slots: idx -1, sqdist +inf.
void orc_knn(const float *map, int m, const float *q, int nq, int k, int *idx, float *sqd, int brute) {
  Cloud c = to_cloud(map, m);
  KdTree t;
  if (!brute) t.setInputCloud(&c);
  for (int i = 0; i < nq; i++) {
    int got = brute ? knn_brute(c, q[i * 4], q[i * 4 + 1], q[i * 4 + 2], k, idx + (size_t)i * k, sqd + (size_t)i * k)
                    : t.nearestKSearch(q[i * 4], q[i * 4 + 1], q[i * 4 + 2], k, idx + (size_t)i * k, sqd + (size_t)i * k);
    for (int j = got; j < k; j++) idx[(size_t)i * k + j] = -1, sqd[(size_t)i * k + j] = INFINITY;
  }
}

// ---- voxel grid; out has capacity n; returns 1 normally, 0 on the int32-overflow copy path
int orc_voxel_grid(const float *in, int n, float leaf, int intensity_last, float *out, int *n_out) {
  Cloud c = to_cloud(in, n), o;
  bool ok = voxel_grid(c, leaf, o, intensity_last != 0);
  *n_out = (int)o.size();
  if (!o.empty()) std::memcpy(out, o.data(), sizeof(PointI) * o.size());
  return ok ? 1 : 0;
}

// ---- extractCloud.  Each out_* has capacity n points; counts = {sharp, less_sharp, flat, less_flat}.
void orc_extract_cloud(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans,
                       float *sharp, float *less_sharp, float *flat, float *less_flat, int *counts, float *curvature,
                       int *label) {
  Cloud c = to_cloud(cloud, n);
  ScanInfo si;
  si.scan_start_ind.assign(scan_start, scan_start + n_scans);
  si.scan_end_ind.assign(scan_end, scan_end + n_scans);
  CloudFeature f;
  extract_cloud(c, si, n_scans, f);
  auto put = [](const Cloud &s, float *dst) {
    if (!s.empty()) std::memcpy(dst, s.data(), sizeof(PointI) * s.size());
    return (int)s.size();
  };
  counts[0] = put(f.corner_points_sharp, sharp);
  counts[1] = put(f.corner_points_less_sharp, less_sharp);
  counts[2] = put(f.surf_points_flat, flat);
  counts[3] = put(f.surf_points_less_flat, less_flat);
  if (curvature) std::memcpy(curvature, f.curvature.data(), sizeof(float) * n);
  if (label) std::memcpy(label, f.label.data(), sizeof(int) * n);
}

// ---- scan-to-map association. type 'c' or 's'. valid[n]; coeffs[n*6]; nn[n*n_neigh] (-1 when invalid)
int orc_match_from_map(int type, const float *map, int m, const float *data, int n, const double *pose7, int n_neigh,
                       int check_fov, const double *opts, unsigned char *valid, double *coeffs, int *nn) {
  Cloud cm = to_cloud(map, m), cd = to_cloud(data, n);
  KdTree t;
  t.setInputCloud(&cm);
  Pose p = to_pose(pose7);
  MatchParams mp = mp_from(opts);
  int cnt = 0;
  for (int i = 0; i < n; i++) {
    Feature f;
    bool ok = type == 'c' ? match_corner_point_from_map(t, cm, cd[i], p, f, i, n_neigh, check_fov != 0, mp)
                          : match_surf_point_from_map(t, cm, cd[i], p, f, i, n_neigh, check_fov != 0, mp);
    valid[i] = ok ? 1 : 0;
    for (int j = 0; j < 6; j++) coeffs[(size_t)i * 6 + j] = ok ? f.coeffs[j] : 0.0;
    if (nn)
      for (int j = 0; j < n_neigh; j++) nn[(size_t)i * n_neigh + j] = ok ? f.nn[j] : -1;
    cnt += ok;
  }
  return cnt;
}

// ---- scan-to-scan association (tracker). type 'c': coeffs 6, 's': coeffs 4. Output compacted in query
// order like the reference: feat_idx[cnt], coeffs[cnt*6], nn3[cnt*3] (nullable: [closest, ind2, ind3], ind3 = -1
// for 'c'). Returns cnt.
int orc_match_from_scan_nn3(int type, const float *scan, int m, const float *data, int n, const double *pose7,
                            const double *opts, int *feat_idx, double *coeffs, int *nn3) {
  Cloud cs = to_cloud(scan, m), cd = to_cloud(data, n);
  KdTree t;
  t.setInputCloud(&cs);
  std::vector<Feature> fs;
  if (type == 'c') match_corner_from_scan(t, cs, cd, to_pose(pose7), fs, mp_from(opts));
  else match_surf_from_scan(t, cs, cd, to_pose(pose7), fs, mp_from(opts));
  for (size_t i = 0; i < fs.size(); i++) {
    feat_idx[i] = (int)fs[i].idx;
    for (int j = 0; j < 6; j++) coeffs[i * 6 + j] = fs[i].coeffs[j];
    if (nn3) nn3[i * 3] = fs[i].nn[0], nn3[i * 3 + 1] = fs[i].nn[1], nn3[i * 3 + 2] = type == 'c' ? -1 : fs[i].nn[2];
  }
  return (int)fs.size();
}
// The same without the neighbour indices (the entry point's original signature, kept for existing callers).
int orc_match_from_scan(int type, const float *scan, int m, const float *data, int n, const double *pose7,
                        const double *opts, int *feat_idx, double *coeffs) {
  return orc_match_from_scan_nn3(type, scan, m, data, n, pose7, opts, feat_idx, coeffs, nullptr);
}

// ---- factors. kind = FactorKind. x = up to 3 parameter blocks (21 doubles). r[3], J[3*21]:
// single-pose kinds write J rows of 7; F_EDGE_VEC writes 3 rows of 7; odom kinds write [Jp|Ji|Je] (21).
void orc_factor_eval(int kind, const double *point3, const double *coeffs6, double sqrt_info, const double *x21,
                     double *r, double *J) {
  V3 p{point3[0], point3[1], point3[2]};
  switch (kind) {
    case F_PLANE: plane_factor(p, coeffs6, sqrt_info, x21, r, J); break;
    case F_EDGE: edge_factor(p, coeffs6, sqrt_info, x21, r, J); break;
    case F_EDGE_VEC: edge_vector_factor(p, coeffs6, x21, r, J); break;
    case F_ODOM_PLANE: odom_plane_factor(p, coeffs6, sqrt_info, x21, x21 + 7, x21 + 14, r, J, J ? J + 7 : nullptr, J ? J + 14 : nullptr); break;
    case F_ODOM_EDGE: odom_edge_factor(p, coeffs6, sqrt_info, x21, x21 + 7, x21 + 14, r, J, J ? J + 7 : nullptr, J ? J + 14 : nullptr); break;
  }
}

// ---- normal equations of a single-pose problem (map factors) at x: features given as SoA.
// types[n] ('s' plane / 'c' edge), points[n*3] double, coeffs[n*6] double. Outputs H36, g6, cost.
void orc_normal_eq(const unsigned char *types, const double *points, const double *coeffs, int n, double sqrt_info,
                   double huber_a, const double *x7, double *H36, double *g6, double *cost) {
  Problem pr;
  pr.huber_a = huber_a;
  double xx[7];
  std::memcpy(xx, x7, sizeof(xx));
  int pid = pr.add_param(xx);
  for (int i = 0; i < n; i++) {
    ResidualBlock b{types[i] == 's' ? F_PLANE : F_EDGE, V3{points[i * 3], points[i * 3 + 1], points[i * 3 + 2]}, {0, 0, 0, 0, 0, 0},
                    sqrt_info, {pid, 0, 0}};
    for (int j = 0; j < 6; j++) b.coeffs[j] = coeffs[(size_t)i * 6 + j];
    pr.blocks.push_back(b);
  }
  NormalEq ne;
  std::vector<const double *> xs{xx};
  pr.evaluate(xs, true, ne);
  std::memcpy(H36, ne.H.data(), 36 * sizeof(double));
  std::memcpy(g6, ne.g.data(), 6 * sizeof(double));
  *cost = ne.cost;
}

// ---- scan2MapOptimization. stats[16]: ran, n_surf, n_corner, lm_iterations, final_cost, degenerate,
// t_kdtree, t_match, t_solver, eig[0..5]
void orc_scan2map(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_scan, int n_ss,
                  const float *corner_scan, int n_cs, const double *pose_init7, const double *opts, double *pose_out7,
                  double *stats, double *H36) {
  Scan2MapOptions o = opts_from(opts);
  o.gf_groups_surf = g_gf_groups_surf, o.gf_groups_corner = g_gf_groups_corner;
  Cloud sm = to_cloud(surf_map, n_sm), cm = to_cloud(corner_map, n_cm), ss = to_cloud(surf_scan, n_ss),
        cs = to_cloud(corner_scan, n_cs);
  Scan2MapResult r = scan2map(sm, cm, ss, cs, to_pose(pose_init7), o);
  pose_to_param(r.pose, pose_out7);
  if (stats) {
    stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
    stats[5] = r.degenerate, stats[6] = r.t_kdtree, stats[7] = r.t_match, stats[8] = r.t_solver;
    for (int i = 0; i < 6; i++) stats[9 + i] = r.eig_last[i];
    stats[15] = 0;
  }
  if (H36) std::memcpy(H36, r.H_last, sizeof(r.H_last));
}

// ---- evalPointUncertainty for a batch: cov6[n*6] float (PointIWithCov::cov_vec layout)
void orc_point_uncertainty(const float *pts, int n, const double *pose7, const double *cov_pose36, const double *cov_meas9, float *cov6) {
  Pose p = to_pose(pose7);
  for (int i = 0; i < n; i++)
    eval_point_uncertainty(PointI{pts[i * 4], pts[i * 4 + 1], pts[i * 4 + 2], pts[i * 4 + 3]}, p, cov_pose36, cov_meas9, cov6 + (size_t)i * 6);
}

// ---- scan2MapOptimization with with_ua = true: per scan point cov_vec (float[6]) -> trace -> sqrt_info clamp
void orc_scan2map_ua(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_scan, int n_ss,
                     const float *surf_cov6, const float *corner_scan, int n_cs, const float *corner_cov6, const double *pose_init7,
                     const double *opts, double *pose_out7, double *stats) {
  Scan2MapOptions o = opts_from(opts);
  std::vector<double> ts(n_ss), tc(n_cs);  // extractCov: float cov_vec -> Matrix3d; trace in double (point_with_cov.hpp:202-214)
  for (int i = 0; i < n_ss; i++) ts[i] = (double)surf_cov6[i * 6] + (double)surf_cov6[i * 6 + 3] + (double)surf_cov6[i * 6 + 5];
  for (int i = 0; i < n_cs; i++) tc[i] = (double)corner_cov6[i * 6] + (double)corner_cov6[i * 6 + 3] + (double)corner_cov6[i * 6 + 5];
  o.surf_cov_trace = &ts, o.corner_cov_trace = &tc;
  Cloud sm = to_cloud(surf_map, n_sm), cm = to_cloud(corner_map, n_cm), ss = to_cloud(surf_scan, n_ss), cs = to_cloud(corner_scan, n_cs);
  Scan2MapResult r = scan2map(sm, cm, ss, cs, to_pose(pose_init7), o);
  pose_to_param(r.pose, pose_out7);
  if (stats) stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
}

// ---- ActiveFeatureSelection::goodFeatureMatching for one feature set (lidar_mapper.h:229-573), explicit seed.
// cov6 nullable (then default_trace).  Outputs: matched[n], jaco[n*6], sel[<= n] (selection order), *n_sel, H[36].
void orc_good_features(int type, const float *map, int m, const float *scan, int n, const float *cov6, double default_trace,
                       const double *pose7, int method, double gf_ratio, unsigned long long seed, int n_neigh, const double *opts,
                       unsigned char *matched, double *jaco, int *sel, int *n_sel, double *H36) {
  Cloud mc = to_cloud(map, m), sc = to_cloud(scan, n);
  KdTree tree;
  tree.setInputCloud(&mc);
  std::vector<double> tr;
  if (cov6) {
    tr.resize(n);
    for (int i = 0; i < n; i++) tr[i] = (double)cov6[i * 6] + (double)cov6[i * 6 + 3] + (double)cov6[i * 6 + 5];
  }
  std::vector<Feature> all;
  std::vector<unsigned char> mt;
  std::vector<double> jc;
  std::vector<int> sl;
  good_feature_matching((char)type, tree, mc, sc, to_pose(pose7), cov6 ? &tr : nullptr, default_trace, method, gf_ratio, seed, n_neigh,
                        opts ? mp_from(opts) : MatchParams(), all, mt, jc, sl, H36);
  for (int i = 0; i < n; i++) matched[i] = mt[i];
  for (size_t i = 0; i < jc.size(); i++) jaco[i] = jc[i];
  for (size_t i = 0; i < sl.size(); i++) sel[i] = sl[i];
  *n_sel = (int)sl.size();
}
// selection only, on caller-provided matched / jaco (kernel-level parity of the selection loop)
void orc_gf_select(int method, double gf_ratio, unsigned long long seed, int n, const unsigned char *matched, const double *jaco,
                   const float *xyz4, int *sel, int *n_sel, double *H36) {
  std::vector<int> sl;
  good_feature_select(method, gf_ratio, seed, n, matched, jaco, xyz4, sl, H36);
  for (size_t i = 0; i < sl.size(); i++) sel[i] = sl[i];
  *n_sel = (int)sl.size();
}

// ---- the whole per-sweep hot path on the CPU: extractCloud -> downsampleCurrentScan -> scan2MapOptimization
// (the bench's cpu_baseline / --impl reference step).  stats[20]: [0..15] as orc_scan2map, [16] t_extract,
// [17] t_downsample, [18] n_surf_in, [19] n_corner_in
void orc_frame(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, const float *surf_map,
               int n_sm, const float *corner_map, int n_cm, float corner_leaf, float surf_leaf, const double *pose_init7,
               const double *opts, double *pose_out7, double *stats) {
  Cloud c = to_cloud(cloud, n);
  ScanInfo si;
  si.scan_start_ind.assign(scan_start, scan_start + n_scans);
  si.scan_end_ind.assign(scan_end, scan_end + n_scans);
  double t0 = now_s();
  CloudFeature f;
  extract_cloud(c, si, n_scans, f);
  double t1 = now_s();
  Cloud cs, ss;
  voxel_grid(f.corner_points_less_sharp, corner_leaf, cs, true);  // lidar_mapper_keyframe.cpp:359-364
  voxel_grid(f.surf_points_less_flat, surf_leaf, ss, true);
  double t2 = now_s();
  double st16[16];
  orc_scan2map(surf_map, n_sm, corner_map, n_cm, ss.empty() ? nullptr : &ss[0].x, (int)ss.size(),
               cs.empty() ? nullptr : &cs[0].x, (int)cs.size(), pose_init7, opts, pose_out7, st16, nullptr);
  if (stats) {
    for (int i = 0; i < 16; i++) stats[i] = st16[i];
    stats[16] = t1 - t0, stats[17] = t2 - t1, stats[18] = (double)ss.size(), stats[19] = (double)cs.size();
  }
}

// ---- the same for a multi-LiDAR frame (odometry node -> mapper hand-over): orc_capi.hpp's prepare_multi, then the mapper's
// scan2MapOptimization on the merged clouds.  ext7: n_lidars x [t q].
// threads > 1: the per-LiDAR extraction under OpenMP like the reference; the mapper part is single-threaded like the reference.

// features of one LiDAR group as they enter scan2MapOptimization (per-LiDAR extractCloud, extrinsic + laser id, merged
// down-sampling); out_* have capacity n points.  Used to restate the sharded (one group per GPU) multi-GPU frame.
void orc_prepare_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                       float corner_leaf, float surf_leaf, float *corner_out, int *n_corner, float *surf_out, int *n_surf) {
  Cloud cs, ss;
  prepare_multi(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, nullptr, 0.f, corner_leaf, surf_leaf, cs, ss, nullptr, nullptr);
  *n_corner = (int)cs.size(), *n_surf = (int)ss.size();
  if (!cs.empty()) std::memcpy(corner_out, cs.data(), sizeof(PointI) * cs.size());
  if (!ss.empty()) std::memcpy(surf_out, ss.data(), sizeof(PointI) * ss.size());
}

// good-feature selection per feature GROUP (one group per GPU in the sharded frame): sizes of the consecutive groups of the
// surf / corner scans of the NEXT orc_scan2map call; n_groups = 0 switches back to one selection over the whole scan.
void orc_set_gf_groups(int n_groups, const int *surf_sizes, const int *corner_sizes) {
  g_gf_groups_surf.assign(surf_sizes, surf_sizes + n_groups);
  g_gf_groups_corner.assign(corner_sizes, corner_sizes + n_groups);
}

void orc_frame_multi(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                     const float *surf_map, int n_sm, const float *corner_map, int n_cm, float corner_leaf, float surf_leaf,
                     const double *pose_init7, const double *opts, double *pose_out7, double *stats) {
  Cloud cs, ss;
  double te = 0, td = 0;
  prepare_multi(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, nullptr, 0.f, corner_leaf, surf_leaf, cs, ss, &te, &td);
  double st16[16];
  orc_scan2map(surf_map, n_sm, corner_map, n_cm, ss.empty() ? nullptr : &ss[0].x, (int)ss.size(),
               cs.empty() ? nullptr : &cs[0].x, (int)cs.size(), pose_init7, opts, pose_out7, st16, nullptr);
  if (stats) {
    for (int i = 0; i < 16; i++) stats[i] = st16[i];
    stats[16] = te, stats[17] = td, stats[18] = (double)ss.size(), stats[19] = (double)cs.size();
  }
}

// ---- online extrinsic calibration step (Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1, estimator.cpp:687-787, with the
// association of buildCalibMap :1135-1149 redone at every outer iteration).  Blocks: pivot (constant, :631), pose_i, ext_ref
// (constant, :642), ext_cal.  Reference LiDAR features of frame i: matched at pivot^-1 * pose_i * ext_ref with n_neigh 5,
// CHECK_FOV true -> LidarPureOdom{PlaneNorm,Edge}Factor(point, coeffs, 1.0) on (pivot, pose_i, ext_ref) (:696-703, :746-754).
// Calibrated LiDAR features at the pivot: matched at ext_cal with n_neigh 10, CHECK_FOV true -> LidarOnlineCalib{PlaneNorm,Edge}Factor
// (point, coeffs, 1.0) on ext_cal (:733-737, :776-779).  HuberLoss(huber_a) (:602), ceres::Solve(max_inner) per outer iteration.
// surf_map_cal / corner_map_cal: the calibrated LiDAR's own local map (leaf 0.2, :1103-1109); n == 0 -> the reference maps.
// stats[4]: lm_iterations, final_cost, residual rows of the last problem, termination
void orc_calib_frame(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_map_cal, int n_smc,
                     const float *corner_map_cal, int n_cmc, const float *surf_ref, int n_sr, const float *corner_ref, int n_cr,
                     const float *surf_cal, int n_sc, const float *corner_cal, int n_cc, const double *pivot7, double *pose_i7,
                     const double *ext_ref7, double *ext_cal7, int max_outer, int max_inner, double huber_a, const double *opts, double *stats) {
  Cloud sm = to_cloud(surf_map, n_sm), cm = to_cloud(corner_map, n_cm), smc = to_cloud(surf_map_cal, n_smc), cmc = to_cloud(corner_map_cal, n_cmc);
  Cloud sr = to_cloud(surf_ref, n_sr), cr = to_cloud(corner_ref, n_cr), sc = to_cloud(surf_cal, n_sc), cc = to_cloud(corner_cal, n_cc);
  KdTree kd_s, kd_c, kd_sc, kd_cc;
  kd_s.setInputCloud(&sm), kd_c.setInputCloud(&cm);
  const bool own = n_smc > 0 && n_cmc > 0;
  if (own) kd_sc.setInputCloud(&smc), kd_cc.setInputCloud(&cmc);
  const MatchParams mp = mp_from(opts);
  double xp[7], xr[7];
  std::memcpy(xp, pivot7, sizeof(xp)), std::memcpy(xr, ext_ref7, sizeof(xr));
  int its = 0, rows = 0, term = 0;
  double cost = 0;
  for (int outer = 0; outer < max_outer; outer++) {
    const Pose pose_a = pose_mul(pose_inv(to_pose(xp)), pose_mul(to_pose(pose_i7), to_pose(xr)));  // :1086-1090
    const Pose pose_b = to_pose(ext_cal7);
    std::vector<Feature> f_sr, f_cr, f_sc, f_cc;
    match_from_map('s', kd_s, sm, sr, pose_a, f_sr, 5, true, mp);
    match_from_map('c', kd_c, cm, cr, pose_a, f_cr, 5, true, mp);
    match_from_map('s', own ? kd_sc : kd_s, own ? smc : sm, sc, pose_b, f_sc, 10, true, mp);
    match_from_map('c', own ? kd_cc : kd_c, own ? cmc : cm, cc, pose_b, f_cc, 10, true, mp);
    Problem pr;
    pr.huber_a = huber_a;
    const int ip = pr.add_param(xp, true), ii = pr.add_param(pose_i7), ir = pr.add_param(xr, true), ie = pr.add_param(ext_cal7);
    for (const Feature &f : f_sr)
      pr.blocks.push_back(ResidualBlock{F_ODOM_PLANE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], 0, 0}, 1.0, {ip, ii, ir}});
    for (const Feature &f : f_sc)
      pr.blocks.push_back(ResidualBlock{F_PLANE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], 0, 0}, 1.0, {ie, 0, 0}});
    for (const Feature &f : f_cr)
      pr.blocks.push_back(ResidualBlock{F_ODOM_EDGE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], f.coeffs[4], f.coeffs[5]}, 1.0, {ip, ii, ir}});
    for (const Feature &f : f_cc)
      pr.blocks.push_back(ResidualBlock{F_EDGE, f.point, {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], f.coeffs[4], f.coeffs[5]}, 1.0, {ie, 0, 0}});
    rows = (int)pr.blocks.size();
    SolveSummary s = solve(pr, max_inner);
    its += s.iterations, cost = s.final_cost, term = s.termination;
  }
  if (stats) stats[0] = its, stats[1] = cost, stats[2] = rows, stats[3] = term;
}

// ---- odometry-side good features (orc_gf.hpp good_feature_matching_odom)
void orc_good_features_odom(int type, const float *map, int m, const float *scan, int n, const double *pivot7, const double *pose_i7, const double *ext7,
                            double gf_ratio, unsigned long long seed, const double *opts, unsigned char *matched, double *jaco, int *sel, int *n_sel,
                            double *H36) {
  Cloud mc = to_cloud(map, m), sc = to_cloud(scan, n);
  KdTree tree;
  tree.setInputCloud(&mc);
  std::vector<Feature> all;
  std::vector<unsigned char> mt;
  std::vector<double> jc;
  std::vector<int> s;
  good_feature_matching_odom((char)type, tree, mc, sc, to_pose(pivot7), to_pose(pose_i7), to_pose(ext7), gf_ratio, seed, mp_from(opts), all, mt, jc, s, H36);
  if (n > 0) std::memcpy(matched, mt.data(), n), std::memcpy(jaco, jc.data(), sizeof(double) * 6 * (size_t)n);
  *n_sel = (int)s.size();
  if (!s.empty()) std::memcpy(sel, s.data(), sizeof(int) * s.size());
}

// ---- Estimator::buildLocalMap / buildCalibMap, the map half (estimator.cpp:1175-1204 / :1084-1110): window clouds -> pivot frame with the
// float matrix of pose_local[i] (pcl::transformPointCloud, PCL 1.8 evaluation order, intensity kept) -> `+=` -> pcl::VoxelGrid(leaf)
void orc_local_map_build(int n_frames, const float *pts, const int *counts, const double *pose_local7, float leaf, float *out, int *n_out) {
  Cloud merged;
  size_t off = 0;
  for (int k = 0; k < n_frames; k++) {
    const FloatTransform xf(pose_local7 + 7 * (size_t)k);
    for (int i = 0; i < counts[k]; i++) {
      const float *p = pts + 4 * (off + i);
      merged.push_back(xf(PointI{p[0], p[1], p[2], p[3]}, p[3]));
    }
    off += (size_t)counts[k];
  }
  Cloud ds;
  voxel_grid(merged, leaf, ds, false);
  *n_out = (int)ds.size();
  if (!ds.empty()) std::memcpy(out, ds.data(), sizeof(PointI) * ds.size());
}

// ---- ImageSegmenter::segmentCloud with segment_flag false: range-image projection + ring re-ordering (orc_segment.hpp)
void orc_project_cloud(const float *cloud, int n, int vertical_scans, int horizon_scans, double roi_range, float *out, int *n_out, int *scan_start,
                       int *scan_end) {
  Cloud c = to_cloud(cloud, n), o;
  std::vector<int> ss, se;
  project_cloud(c, vertical_scans, horizon_scans, roi_range, o, ss, se);
  *n_out = (int)o.size();
  if (!o.empty()) std::memcpy(out, o.data(), sizeof(PointI) * o.size());
  std::memcpy(scan_start, ss.data(), sizeof(int) * vertical_scans), std::memcpy(scan_end, se.data(), sizeof(int) * vertical_scans);
}

// pixel (row * horizon_scans + column) of every point, -1 where projectCloud skips it before the first-point-wins test
void orc_project_pixels(const float *cloud, int n, int vertical_scans, int horizon_scans, double roi_range, int *pix) {
  const SegmenterParam sp = segmenter_param(vertical_scans, horizon_scans);
  for (int i = 0; i < n; i++) {
    PointI p;
    p.x = cloud[4 * i], p.y = cloud[4 * i + 1], p.z = cloud[4 * i + 2], p.intensity = cloud[4 * i + 3];
    int row, col;
    float range;
    pix[i] = project_point(sp, p, roi_range, &row, &col, &range) ? row * horizon_scans + col : -1;
  }
}

// ---- submap assembly with uncertainty (orc_uct.hpp)
void orc_compound_pose_cov(const double *p1, const double *cov1, const double *p2, const double *cov2, double *pose_out7, double *cov_out36) {
  M6 c1, c2, cc;
  std::memcpy(c1.m, cov1, sizeof(c1.m)), std::memcpy(c2.m, cov2, sizeof(c2.m));
  // the reference's Pose objects are normalised on construction; the product is not re-normalised (associate_uct.hpp:37-38)
  const Pose a = to_pose(p1), b = to_pose(p2);
  Pose pc;
  compound_pose_with_cov(a, c1, b, c2, pc, cc);
  pose_to_param(pc, pose_out7);
  std::memcpy(cov_out36, cc.m, sizeof(cc.m));
}
// cloud: [n,4] (intensity = laser id); ext7 / pose_compound7: n_lasers x 7; cov_compound: n_lasers x 36.  out_*: capacity n.
void orc_cloud_uct_associate(const float *cloud, int n, const double *pose_global7, int n_lasers, const double *ext7, const double *pose_compound7,
                             const double *cov_compound36, const double *cov_meas9, int with_ua, double trace_threshold, float *out_pts,
                             float *out_cov6, float *out_trace, int *n_out) {
  Cloud c = to_cloud(cloud, n);
  std::vector<Pose> pe, pc;
  std::vector<M6> cc(n_lasers);
  for (int l = 0; l < n_lasers; l++) {
    pe.push_back(to_pose(ext7 + 7 * l)), pc.push_back(to_pose(pose_compound7 + 7 * l));
    std::memcpy(cc[l].m, cov_compound36 + 36 * l, sizeof(cc[l].m));
  }
  CovCloud o;
  cloud_uct_associate(c, to_pose(pose_global7), pe, pc, cc, cov_meas9, with_ua != 0, trace_threshold, o);
  *n_out = (int)o.pts.size();
  if (*n_out) {
    std::memcpy(out_pts, o.pts.data(), sizeof(PointI) * o.pts.size());
    std::memcpy(out_cov6, o.cov6.data(), sizeof(float) * o.cov6.size());
    std::memcpy(out_trace, o.trace.data(), sizeof(float) * o.trace.size());
  }
}
int orc_voxel_grid_cov(const float *pts, const float *cov6, const float *trace, int n, float leaf, float trace_threshold, float *out_pts, float *out_cov6,
                       float *out_trace, int *n_out) {
  CovCloud in, o;
  in.pts = to_cloud(pts, n);
  in.cov6.assign(cov6, cov6 + 6 * (size_t)n), in.trace.assign(trace, trace + n);
  const bool ok = voxel_grid_cov(in, leaf, trace_threshold, o);
  *n_out = (int)o.pts.size();
  if (*n_out) {
    std::memcpy(out_pts, o.pts.data(), sizeof(PointI) * o.pts.size());
    std::memcpy(out_cov6, o.cov6.data(), sizeof(float) * o.cov6.size());
    std::memcpy(out_trace, o.trace.data(), sizeof(float) * o.trace.size());
  }
  return ok ? 1 : 0;
}

// ---- Estimator::optimizeMap residual blocks for one frame / one LiDAR (estimator.cpp:687-848): LidarPureOdom factors on
// (pose_pivot [constant], pose_i, ext_n); free_mask bit 0 frees pose_i, bit 1 frees ext.  ceres::Solve(max_it),
// HuberLoss(huber_a).  stats[3]: lm_iterations, final_cost, termination
void orc_odom_solve(int n, const unsigned char *types, const double *points, const double *coeffs, const double *pivot7,
                    double *pose_i7, double *ext7, int free_mask, int max_it, double huber_a, double sqrt_info, double *stats) {
  Problem pr;
  pr.huber_a = huber_a;
  double xp[7];
  std::memcpy(xp, pivot7, sizeof(xp));
  int ip = pr.add_param(xp, true);  // SetParameterBlockConstant(para_pose_[0]), estimator.cpp:631
  int ii = pr.add_param(pose_i7, !(free_mask & 1));
  int ie = pr.add_param(ext7, !(free_mask & 2));
  for (int i = 0; i < n; i++) {
    ResidualBlock b{types[i] == 's' ? F_ODOM_PLANE : F_ODOM_EDGE, V3{points[i * 3], points[i * 3 + 1], points[i * 3 + 2]},
                    {0, 0, 0, 0, 0, 0}, sqrt_info, {ip, ii, ie}};
    for (int j = 0; j < 6; j++) b.coeffs[j] = coeffs[(size_t)i * 6 + j];
    pr.blocks.push_back(b);
  }
  SolveSummary s = solve(pr, max_it);
  if (stats) stats[0] = s.iterations, stats[1] = s.final_cost, stats[2] = s.termination;
}

// ---- LidarTracker::trackCloud. stats[3]: n_corner, n_surf, lm_iterations
void orc_track_cloud(const float *prev_less_sharp, int n_pls, const float *prev_less_flat, int n_plf,
                     const float *cur_sharp, int n_cs, const float *cur_flat, int n_cf, const double *pose_ini7,
                     const double *opts, double *pose_out7, double *stats) {
  TrackOptions o;
  o.max_outer = (int)opts[O_MAX_OUTER], o.max_inner = (int)opts[O_MAX_INNER], o.huber_a = opts[O_HUBER];
  o.mp = mp_from(opts);
  Cloud a = to_cloud(prev_less_sharp, n_pls), b = to_cloud(prev_less_flat, n_plf), c = to_cloud(cur_sharp, n_cs),
        d = to_cloud(cur_flat, n_cf);
  TrackResult r = track_cloud(a, b, c, d, to_pose(pose_ini7), o);
  pose_to_param(r.pose, pose_out7);
  if (stats) stats[0] = r.n_corner, stats[1] = r.n_surf, stats[2] = r.lm_iterations;
}

// ---- TransformToEnd (orc_capi.hpp) of n points (x y z intensity) with one pose [t q]
void orc_undist_points(const float *pts, int n, const double *pose7, float scan_period, float *out) {
  Cloud c = to_cloud(pts, n);
  undistort_cloud(c, pose7, scan_period);
  if (n > 0) std::memcpy(out, c.data(), sizeof(PointI) * (size_t)n);
}

// pose_undist of every LiDAR (out7: n_lidars x 7): Estimator::process, estimator.cpp:575-579, pose_undist[n] =
// Pose(qbl_n, tbl_n).inverse() * pose_rlt_[IDX_REF] * Pose(qbl_n, tbl_n); every LiDAR takes IDX_REF's unless ESTIMATE_EXTRINSIC == 2
void orc_undist_poses(const double *rlt7, int idx_ref, int n_lidars, const double *ext7, int estimate_extrinsic, double *out7) {
  const Pose rlt = to_pose(rlt7);
  std::vector<Pose> und(n_lidars);
  for (int n = 0; n < n_lidars; n++) {
    const double *e = ext7 + 7 * n;
    const Pose ext = make_pose(Q4{e[3], e[4], e[5], e[6]}, V3{e[0], e[1], e[2]});
    const Q4 &q = ext.q;  // Pose::inverse = Pose(q.inverse(), -(q.inverse() * t)), Quaternion::inverse = conj / squaredNorm
    const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
    const Q4 qi{-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
    und[n] = pose_mul(pose_mul(make_pose(qi, -qrot(qi, ext.t)), rlt), ext);
  }
  for (int n = 0; n < n_lidars; n++) pose_to_param(und[estimate_extrinsic == 2 ? n : idx_ref], out7 + 7 * n);
}

// OpenMP threads used by the parallel sections (1 = the reference's serial behaviour; tests always use 1).
void orc_set_threads(int n) {
#ifdef _OPENMP
  omp_set_num_threads(n < 1 ? 1 : n);
#else
  (void)n;
#endif
}

int orc_max_threads() {
#ifdef _OPENMP
  return omp_get_max_threads();
#else
  return 1;
#endif
}

}  // extern "C"
