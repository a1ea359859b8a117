// ORACLE — TEST INFRASTRUCTURE ONLY (see oracle/orc_math.hpp's header).
// The DISTORTION step of the odometry restated over the oracle's frame (oracle/orc_ua.cpp, included whole):
//   Estimator::process              estimator.cpp:575-579: pose_undist[n] = Pose(qbl_n, tbl_n).inverse() * pose_rlt_[IDX_REF] * Pose(qbl_n, tbl_n)
//                                   (Pose::inverse / operator*, pose.cpp:99-113, every Pose normalising its quaternion)
//   undistortMeasurements           :376-408: corner_points_less_sharp and surf_points_less_flat of LiDAR n moved with pose_undist[n] when
//                                   ESTIMATE_EXTRINSIC == 2, else with pose_undist[IDX_REF]; sharp, flat and the outlier cloud untouched
//   TransformToEnd                  utility.h:54-100 with Eigen 3.3's slerp (Identity.slerp(s, q): d = q.w, acos / sin of the C library,
//                                   weights 1 - s and s when |d| >= 1 - DBL_EPSILON, the second weight negated when d < 0, the coefficients
//                                   scale0 (0,0,0,1) + scale1 q NOT renormalised), _transformVector, Quaternion::inverse = conj / squaredNorm
//   the frame                       orc_frame_multi / orc_ua_frame_multi with the step between each LiDAR's extractCloud and
//                                   transformCloudFeature; or, without the rig merge, the whole sweep's extractCloud, the step, and
//                                   pointAssociateToMap with the single extrinsic (mloam_set_extrinsic)
// Restatement choices (in addition to orc_math.hpp's and orc_ua.cpp's):
//   - squaredNorm and normalize sum x, y, z, w in order (orc_math.hpp qnormalized);
//   - s = (float)(intensity - (float)int(intensity)) / (float)scan_period, as the float expression of utility.h:64, widened to double.
#include "../../oracle/orc_ua.cpp"

#include <cfloat>

namespace {

// TransformToEnd(p, p, pose, true, scan_period), pose as given (a Pose holds a normalised q)
PointI transform_to_end(const PointI &p, const Pose &pose, float scan_period) {
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

Pose pose_inverse_eigen(const Pose &a) {  // Pose(q.inverse(), -(q.inverse() * t))
  const double n2 = a.q.x * a.q.x + a.q.y * a.q.y + a.q.z * a.q.z + a.q.w * a.q.w;
  const Q4 qi{-a.q.x / n2, -a.q.y / n2, -a.q.z / n2, a.q.w / n2};
  return make_pose(qi, -qrot(qi, a.t));
}

void undistort_poses(const double *rlt7, int idx_ref, int n_lidars, const double *ext7, int estimate_extrinsic, double *out7) {
  const Pose rlt = to_pose(rlt7);
  std::vector<Pose> und(n_lidars);
  for (int n = 0; n < n_lidars; n++) {
    const double *e = ext7 + 7 * n;
    const Pose ext = make_pose(Q4{e[3], e[4], e[5], e[6]}, V3{e[0], e[1], e[2]});
    und[n] = pose_mul(pose_mul(pose_inverse_eigen(ext), rlt), ext);
  }
  for (int n = 0; n < n_lidars; n++) pose_to_param(und[estimate_extrinsic == 2 ? n : idx_ref], out7 + 7 * n);
}

void undistort(Cloud &c, const double *pose7, float scan_period) {
  const Pose p = to_pose(pose7);
  for (PointI &q : c) q = transform_to_end(q, p, scan_period);
}

// The features entering downsampleCurrentScan's filters and the filtered scans.  ext7 (n_lidars x 7): the rig merge; nullptr: the whole
// sweep is one LiDAR's, moved with single_ext7 (nullable) by pointAssociateToMap.  poses7 (nullable): the undistortion, one pose per LiDAR.
void prepare(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
             const double *single_ext7, const double *poses7, float scan_period, float corner_leaf, float surf_leaf, Cloud &cs, Cloud &ss) {
  Cloud corner, surf;
  if (!ext7) {
    CloudFeature f;
    ScanInfo si;
    si.scan_start_ind.assign(scan_start, scan_start + n_scans), si.scan_end_ind.assign(scan_end, scan_end + n_scans);
    extract_cloud(to_cloud(cloud, n), si, n_scans, f);
    corner = f.corner_points_less_sharp, surf = f.surf_points_less_flat;
    if (poses7) undistort(corner, poses7, scan_period), undistort(surf, poses7, scan_period);
    if (single_ext7) {
      const Pose T = to_pose(single_ext7);
      for (PointI &p : corner) p = associate(p, T);
      for (PointI &p : surf) p = associate(p, T);
    }
  } else {
    const int R = n_scans / n_lidars;
    for (int l = 0; l < n_lidars; l++) {
      const int lo = scan_start[l * R] - 5, hi = (l + 1 < n_lidars) ? scan_start[(l + 1) * R] - 5 : n;
      Cloud c = to_cloud(cloud + 4 * (size_t)lo, hi - lo);
      ScanInfo si;
      for (int r = 0; r < R; r++) si.scan_start_ind.push_back(scan_start[l * R + r] - lo), si.scan_end_ind.push_back(scan_end[l * R + r] - lo);
      CloudFeature f;
      extract_cloud(c, si, R, f);
      if (poses7) undistort(f.corner_points_less_sharp, poses7 + 7 * l, scan_period), undistort(f.surf_points_less_flat, poses7 + 7 * l, scan_period);
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
      xf(f.corner_points_less_sharp, corner);
      xf(f.surf_points_less_flat, surf);
    }
  }
  voxel_grid(corner, corner_leaf, cs, true);
  voxel_grid(surf, surf_leaf, ss, true);
}

}  // namespace

extern "C" {

// TransformToEnd of n points (x y z intensity) with one pose [t q]
void orc_undist_points(const float *pts, int n, const double *pose7, float scan_period, float *out) {
  Cloud c = to_cloud(pts, n);
  undistort(c, pose7, scan_period);
  if (n > 0) std::memcpy(out, c.data(), sizeof(PointI) * (size_t)n);
}

void orc_undist_poses(const double *rlt7, int idx_ref, int n_lidars, const double *ext7, int estimate_extrinsic, double *out7) {
  undistort_poses(rlt7, idx_ref, n_lidars, ext7, estimate_extrinsic, out7);
}

// A frame with the undistortion: as orc_frame_multi (ext_cov36 == nullptr) or orc_ua_frame_multi (with_ua; ext7 required), ext7 / single_ext7
// / poses7 as prepare.  stats[20] as orc_ua_frame_multi; the scans entering the solve (gated with with_ua), capacity n each, with cov_vec.
void orc_undist_frame(const float *cloud, int n, const int *scan_start, const int *scan_end, int n_scans, int n_lidars, const double *ext7,
                      const double *single_ext7, const double *poses7, float scan_period, const double *ext_cov36, const double *cov_meas9,
                      double trace_threshold, const float *surf_map, int n_sm, const float *corner_map, int n_cm, float corner_leaf,
                      float surf_leaf, const double *pose_init7, const double *opts, double *pose_out7, double *stats, double *cov36,
                      float *surf_out, float *surf_cov6, int *n_surf, float *corner_out, float *corner_cov6, int *n_corner) {
  Cloud cs, ss;
  prepare(cloud, n, scan_start, scan_end, n_scans, n_lidars, ext7, single_ext7, poses7, scan_period, corner_leaf, surf_leaf, cs, ss);
  const bool with_ua = ext_cov36 != nullptr;
  Cloud sg, cg;
  std::vector<float> sc6, cc6;
  std::vector<double> st, ct;
  auto gate = [&](const Cloud &in, Cloud &out, std::vector<float> &cov6, std::vector<double> &tr) {
    for (const PointI &p : in) {
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
      tr.push_back((double)c6[0] + (double)c6[3] + (double)c6[5]);
    }
  };
  gate(ss, sg, sc6, st);
  gate(cs, cg, cc6, ct);
  Scan2MapOptions o = opts_from(opts);
  double cov[36] = {0}, H[36];
  Scan2MapResult r;
  if (with_ua) {
    o.surf_cov_trace = &st, o.corner_cov_trace = &ct;
    r = scan2map_with_cov(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), sg, cg, to_pose(pose_init7), o, cov, H);
  } else {
    r = scan2map(to_cloud(surf_map, n_sm), to_cloud(corner_map, n_cm), sg, cg, to_pose(pose_init7), o);
  }
  pose_to_param(r.pose, pose_out7);
  for (int i = 0; i < 20; i++) stats[i] = 0;
  stats[0] = r.ran, stats[1] = r.n_surf, stats[2] = r.n_corner, stats[3] = r.lm_iterations, stats[4] = r.final_cost;
  stats[5] = r.degenerate;
  for (int i = 0; i < 6; i++) stats[9 + i] = r.eig_last[i];
  stats[18] = (double)sg.size(), stats[19] = (double)cg.size();
  if (cov36) std::memcpy(cov36, cov, sizeof(cov));
  *n_surf = (int)sg.size(), *n_corner = (int)cg.size();
  if (!sg.empty()) std::memcpy(surf_out, sg.data(), sizeof(PointI) * sg.size()), std::memcpy(surf_cov6, sc6.data(), sizeof(float) * sc6.size());
  if (!cg.empty()) std::memcpy(corner_out, cg.data(), sizeof(PointI) * cg.size()), std::memcpy(corner_cov6, cc6.data(), sizeof(float) * cc6.size());
}

}  // extern "C"
