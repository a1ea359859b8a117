// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).
// The online-calibration step over the whole rig (Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1, estimator.cpp:633-642,
// 670-787, NUM_OF_LASER = L): orc_calib_frame's association and factors for every LiDAR, every non-reference extrinsic free in one
// problem, and with prior_factor: 1 a PriorFactor (prior_factor.hpp:27-72) on every extrinsic (:675-685), the constant ext_ref's
// included.  The LM is orc_solver.hpp's ceres::Solve restatement with the prior residual blocks added to each evaluation; without
// priors it performs solve()'s arithmetic, so L = 2 equals orc_calib_frame bit for bit.
#include "orc_capi.hpp"

using namespace orc;

namespace {

// PriorFactor::Evaluate (prior_factor.hpp:36-71): residual = sqrt_info [P - pos_ ; 2 (rot_^-1 Q).vec], sqrt_info = diag(sp I3, sr I3);
// local jacobian = sqrt_info diag(I3, LeftQuatMatrix(Q^-1 rot_).topLeftCorner<3,3>()) as written (the reference marks its rotation
// block "seem to be wrong").  Eigen's Quaternion::inverse() is conjugate / squaredNorm.
Q4 qinv(const Q4 &q) {
  const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
}
void prior_factor(const double *x, const double *x0, double sp, double sr, double r[6], double J[36]) {
  const Q4 Q{x[3], x[4], x[5], x[6]}, R0{x0[3], x0[4], x0[5], x0[6]};
  const Q4 e = qmul(qinv(R0), Q);
  r[0] = sp * (x[0] - x0[0]), r[1] = sp * (x[1] - x0[1]), r[2] = sp * (x[2] - x0[2]);
  r[3] = sr * (2 * e.x), r[4] = sr * (2 * e.y), r[5] = sr * (2 * e.z);
  if (!J) return;
  const Q4 m = qmul(qinv(Q), R0);
  const double L[9] = {m.w, -m.z, m.y, m.z, m.w, -m.x, -m.y, m.x, m.w};  // w I + [v]x
  for (int k = 0; k < 36; k++) J[k] = 0.0;
  for (int k = 0; k < 3; k++) J[k * 6 + k] = sp;
  for (int i = 0; i < 3; i++)
    for (int j = 0; j < 3; j++) J[(3 + i) * 6 + 3 + j] = sr * L[i * 3 + j];
}

struct Prior {
  int pb;            // parameter block
  const double *x0;  // tbl_ / qbl_
};

// Problem::evaluate + the prior blocks (no loss)
void evaluate(const Problem &prob, const std::vector<Prior> &priors, double sp, double sr, const std::vector<const double *> &xs, bool want_jac,
              NormalEq &ne) {
  prob.evaluate(xs, want_jac, ne);
  const std::vector<int> off = prob.offsets();
  for (const Prior &p : priors) {
    double r[6], J[36];
    prior_factor(xs[p.pb], p.x0, sp, sr, r, want_jac ? J : nullptr);
    double s = 0;
    for (int i = 0; i < 6; i++) s += r[i] * r[i];
    ne.cost += 0.5 * s;
    const int o = off[p.pb];
    if (!want_jac || o < 0) continue;
    for (int i = 0; i < 6; i++)
      for (int a = 0; a < 6; a++) {
        ne.g[o + a] += J[i * 6 + a] * r[i];
        for (int c = 0; c < 6; c++) ne.H[(size_t)(o + a) * ne.n + o + c] += J[i * 6 + a] * J[i * 6 + c];
      }
  }
}

// orc_solver.hpp solve() with evaluate() above (same statements, same order)
SolveSummary solve_rig(Problem &prob, const std::vector<Prior> &priors, double sp, double sr, int max_num_iterations) {
  SolveSummary sum;
  int n;
  std::vector<int> off = prob.offsets(&n);
  const size_t nb = prob.params.size();
  std::vector<std::vector<double>> x(nb, std::vector<double>(7)), xc(nb, std::vector<double>(7));
  for (size_t i = 0; i < nb; i++) std::memcpy(x[i].data(), prob.params[i], 7 * sizeof(double));
  auto ptrs = [&](std::vector<std::vector<double>> &v) {
    std::vector<const double *> p(nb);
    for (size_t i = 0; i < nb; i++) p[i] = v[i].data();
    return p;
  };
  auto xnorm = [&](std::vector<std::vector<double>> &v) {
    double s = 0;
    for (size_t i = 0; i < nb; i++)
      if (!prob.constant[i])
        for (int k = 0; k < 7; k++) s += v[i][k] * v[i][k];
    return std::sqrt(s);
  };
  auto plus = [&](std::vector<std::vector<double>> &from, const std::vector<double> &delta, std::vector<std::vector<double>> &to) {
    for (size_t i = 0; i < nb; i++) {
      if (off[i] < 0) to[i] = from[i];
      else prob.local[i].Plus(from[i].data(), &delta[off[i]], to[i].data());
    }
  };
  const double min_diag = 1e-6, max_diag = 1e32, max_radius = 1e16;
  const double function_tolerance = 1e-6, parameter_tolerance = 1e-8, gradient_tolerance = 1e-10;
  const double min_relative_decrease = 1e-3;
  double radius = 1e4, decrease_factor = 2.0;
  bool reuse_diagonal = false;
  NormalEq ne;
  evaluate(prob, priors, sp, sr, ptrs(x), true, ne);
  double cost = ne.cost;
  sum.initial_cost = sum.final_cost = cost;
  if (n == 0) return sum;
  double x_norm = xnorm(x);
  std::vector<double> scale(n), diag(n), lmd(n), step(n), delta(n), Hs((size_t)n * n), gs(n);
  for (int j = 0; j < n; j++) scale[j] = 1.0 / (1.0 + std::sqrt(ne.H[(size_t)j * n + j]));
  auto gradient_max_norm = [&]() {
    std::vector<double> neg(n);
    for (int j = 0; j < n; j++) neg[j] = -ne.g[j];
    plus(x, neg, xc);
    double m = 0;
    for (size_t i = 0; i < nb; i++)
      if (off[i] >= 0)
        for (int k = 0; k < 7; k++) m = std::max(m, std::fabs(x[i][k] - xc[i][k]));
    return m;
  };
  if (gradient_max_norm() <= gradient_tolerance) {
    sum.termination = 3;
    return sum;
  }
  int num_consecutive_invalid = 0, iteration = 0;
  while (true) {
    if (iteration >= max_num_iterations) {
      sum.termination = 0;
      break;
    }
    for (int a = 0; a < n; a++) {
      gs[a] = scale[a] * ne.g[a];
      for (int b = 0; b < n; b++) Hs[(size_t)a * n + b] = scale[a] * ne.H[(size_t)a * n + b] * scale[b];
    }
    if (!reuse_diagonal)
      for (int j = 0; j < n; j++) diag[j] = std::min(std::max(Hs[(size_t)j * n + j], min_diag), max_diag);
    for (int j = 0; j < n; j++) lmd[j] = std::sqrt(diag[j] / radius);
    std::vector<double> A(Hs);
    for (int j = 0; j < n; j++) A[(size_t)j * n + j] += lmd[j] * lmd[j];
    bool ok = cholesky(n, A.data());
    if (ok) {
      cholesky_solve(n, A.data(), gs.data(), step.data());
      for (int j = 0; j < n; j++) {
        step[j] = -step[j];
        if (!std::isfinite(step[j])) ok = false;
      }
    }
    reuse_diagonal = true;
    iteration++;
    sum.iterations = iteration;
    double model_cost_change = 0;
    if (ok) {
      double sg = 0, sHs = 0;
      for (int a = 0; a < n; a++) {
        sg += step[a] * gs[a];
        double t = 0;
        for (int b = 0; b < n; b++) t += Hs[(size_t)a * n + b] * step[b];
        sHs += step[a] * t;
      }
      model_cost_change = -(sg + 0.5 * sHs);
      if (model_cost_change < 0) ok = false;
    }
    if (!ok) {
      if (++num_consecutive_invalid >= 5) {
        sum.termination = 4;
        break;
      }
      radius *= 0.5;
      reuse_diagonal = true;
      continue;
    }
    num_consecutive_invalid = 0;
    for (int j = 0; j < n; j++) delta[j] = step[j] * scale[j];
    plus(x, delta, xc);
    NormalEq nc;
    evaluate(prob, priors, sp, sr, ptrs(xc), false, nc);
    const double new_cost = nc.cost;
    double step_norm = 0;
    for (size_t i = 0; i < nb; i++)
      if (off[i] >= 0)
        for (int k = 0; k < 7; k++) step_norm += (x[i][k] - xc[i][k]) * (x[i][k] - xc[i][k]);
    step_norm = std::sqrt(step_norm);
    if (step_norm <= parameter_tolerance * (x_norm + parameter_tolerance)) {
      sum.termination = 2;
      break;
    }
    const double cost_change = cost - new_cost;
    if (std::fabs(cost_change) <= function_tolerance * cost) {
      sum.termination = 1;
      break;
    }
    const double relative_decrease = cost_change / model_cost_change;
    if (relative_decrease > min_relative_decrease) {
      sum.successful++;
      radius = radius / std::max(1.0 / 3.0, 1.0 - std::pow(2.0 * relative_decrease - 1.0, 3));
      radius = std::min(max_radius, radius);
      decrease_factor = 2.0;
      reuse_diagonal = false;
      x = xc;
      x_norm = xnorm(x);
      evaluate(prob, priors, sp, sr, ptrs(x), true, ne);
      cost = ne.cost;
      if (gradient_max_norm() <= gradient_tolerance) {
        sum.termination = 3;
        break;
      }
    } else {
      radius = radius / decrease_factor;
      decrease_factor *= 2.0;
      reuse_diagonal = true;
    }
  }
  sum.final_cost = cost;
  for (size_t i = 0; i < nb; i++)
    if (!prob.constant[i]) std::memcpy(prob.params[i], x[i].data(), 7 * sizeof(double));
  return sum;
}

}  // namespace

extern "C" {

// r[6], J[36] (row-major, local 6x6) of PriorFactor at x7 with target x07
void orc_prior_factor(const double *x7, const double *x07, double pos_scale, double rot_scale, double *r6, double *J36) {
  prior_factor(x7, x07, pos_scale, rot_scale, r6, J36);
}

// surf / corner: L clouds concatenated in LiDAR order (counts per LiDAR).  Cloud idx_ref: frame i's features at pivot^-1 * pose_i *
// ext_ref (n_neigh 5) -> LidarPureOdom* on pose_i; cloud n != idx_ref at ext7s[n] (n_neigh 10, against surf_map_cal / corner_map_cal when
// both are non-empty) -> LidarOnlineCalib* on ext7s[n].  CHECK_FOV true.  prior_pos = prior_rot = 0: no priors.
// stats[4]: lm_iterations, final_cost, feature rows of the last problem, termination; rows[L]: feature rows per LiDAR.
void orc_calib_rig(const float *surf_map, int n_sm, const float *corner_map, int n_cm, const float *surf_map_cal, int n_smc,
                   const float *corner_map_cal, int n_cmc, int L, int idx_ref, const float *surf, const int *surf_counts, const float *corner,
                   const int *corner_counts, const double *pivot7, double *pose_i7, double *ext7s, const double *prior7s, double prior_pos,
                   double prior_rot, int max_outer, int max_inner, double huber_a, const double *opts, double *stats, int *rows) {
  Cloud sm = to_cloud(surf_map, n_sm), cm = to_cloud(corner_map, n_cm), smc = to_cloud(surf_map_cal, n_smc), cmc = to_cloud(corner_map_cal, n_cmc);
  std::vector<Cloud> sc(L), cc(L);
  for (int n = 0, os = 0, oc = 0; n < L; n++) {
    sc[n] = to_cloud(surf + 4 * (size_t)os, surf_counts[n]), cc[n] = to_cloud(corner + 4 * (size_t)oc, corner_counts[n]);
    os += surf_counts[n], oc += corner_counts[n];
  }
  KdTree kd_s, kd_c, kd_sc, kd_cc;
  kd_s.setInputCloud(&sm), kd_c.setInputCloud(&cm);
  const bool own = n_smc > 0 && n_cmc > 0;
  if (own) kd_sc.setInputCloud(&smc), kd_cc.setInputCloud(&cmc);
  const MatchParams mp = mp_from(opts);
  const bool has_prior = prior_pos != 0.0 || prior_rot != 0.0;
  double xp[7], xr[7];
  std::memcpy(xp, pivot7, sizeof(xp)), std::memcpy(xr, ext7s + 7 * idx_ref, sizeof(xr));
  int its = 0, term = 0, total = 0;
  double cost = 0;
  std::vector<int> nrows(L, 0);
  for (int outer = 0; outer < max_outer; outer++) {
    std::vector<std::vector<Feature>> fs(L), fc(L);
    const Pose pose_a = pose_mul(pose_inv(to_pose(xp)), pose_mul(to_pose(pose_i7), to_pose(xr)));  // :1086-1090
    for (int n = 0; n < L; n++) {
      if (n == idx_ref) {
        match_from_map('s', kd_s, sm, sc[n], pose_a, fs[n], 5, true, mp);
        match_from_map('c', kd_c, cm, cc[n], pose_a, fc[n], 5, true, mp);
      } else {
        const Pose pose_b = to_pose(ext7s + 7 * n);
        match_from_map('s', own ? kd_sc : kd_s, own ? smc : sm, sc[n], pose_b, fs[n], 10, true, mp);
        match_from_map('c', own ? kd_cc : kd_c, own ? cmc : cm, cc[n], pose_b, fc[n], 10, true, mp);
      }
    }
    Problem pr;
    pr.huber_a = huber_a;
    const int ip = pr.add_param(xp, true), ii = pr.add_param(pose_i7), ir = pr.add_param(xr, true);
    std::vector<int> ie(L, ir);
    for (int n = 0; n < L; n++)
      if (n != idx_ref) ie[n] = pr.add_param(ext7s + 7 * n);
    // orc_calib_frame's block order: surf of the reference LiDAR, surf of the calibrated ones, then the corners likewise
    for (int t = 0; t < 2; t++) {
      const std::vector<std::vector<Feature>> &F = t == 0 ? fs : fc;
      for (const Feature &f : F[idx_ref])
        pr.blocks.push_back(ResidualBlock{t == 0 ? F_ODOM_PLANE : F_ODOM_EDGE, f.point,
                                          {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], t == 0 ? 0 : f.coeffs[4], t == 0 ? 0 : f.coeffs[5]}, 1.0, {ip, ii, ir}});
      for (int n = 0; n < L; n++)
        if (n != idx_ref)
          for (const Feature &f : F[n])
            pr.blocks.push_back(ResidualBlock{t == 0 ? F_PLANE : F_EDGE, f.point,
                                              {f.coeffs[0], f.coeffs[1], f.coeffs[2], f.coeffs[3], t == 0 ? 0 : f.coeffs[4], t == 0 ? 0 : f.coeffs[5]}, 1.0, {ie[n], 0, 0}});
    }
    std::vector<Prior> priors;
    if (has_prior)
      for (int n = 0; n < L; n++) priors.push_back(Prior{ie[n], prior7s + 7 * n});  // ie[idx_ref] = ir: the constant ext_ref
    total = (int)pr.blocks.size();
    for (int n = 0; n < L; n++) nrows[n] = (int)(fs[n].size() + fc[n].size());
    SolveSummary s = solve_rig(pr, priors, prior_pos, prior_rot, max_inner);
    its += s.iterations, cost = s.final_cost, term = s.termination;
  }
  if (stats) stats[0] = its, stats[1] = cost, stats[2] = total, stats[3] = term;
  if (rows)
    for (int n = 0; n < L; n++) rows[n] = nrows[n];
}

}  // extern "C"
