// lm.cuh — the one statement of the trust-region policy every device solve follows: Ceres 1.12's TrustRegionMinimizer with the
// LevenbergMarquardtStrategy and DENSE_QR/DENSE_SCHUR defaults the reference never overrides (SURVEY.md §8c).
//
//   constants        the Ceres defaults, once
//   LMTermination    the values of mloam_solve_stats_t::termination
//   chol / chol6     the Cholesky factors of the damped systems
//   lm_*             the policy's rules as pure helpers: LM diagonal clamp, verdict on an evaluated step, radius updates.  The pose
//                    warp tail (solve_kernels.cu) and the rig's one-lane-per-block machine (calib_rig.cu) call them.
//   lm_begin /       the single-thread state machine (ComputeStep with the invalid-step loop, then the step's verdict), on a problem type:
//   lm_digest        the pose (solve_kernels.cu, MLOAM_LM_TAIL=serial) and the odometry's 6 / 12-DoF chain (odom_kernels.cu).
#pragma once

namespace mloam {

// Ceres defaults the reference relies on (never overridden in-tree; SURVEY.md §8c)
__device__ constexpr double kMinDiag = 1e-6, kMaxDiag = 1e32, kMaxRadius = 1e16, kInitialRadius = 1e4, kDecreaseFactor = 2.0;
__device__ constexpr double kFuncTol = 1e-6, kParamTol = 1e-8, kGradTol = 1e-10, kMinRelDecrease = 1e-3;
constexpr int kMaxInvalidSteps = 5;

// mloam_solve_stats_t::termination (public: the values do not change)
enum LMTermination : int {
  kTermMaxIterations = 0,
  kTermFunctionTol = 1,
  kTermParameterTol = 2,
  kTermGradientTol = 3,
  kTermInvalidSteps = 4,   // five steps in a row did not factor, were not finite or did not decrease the model
  kTermTooFewRows = 5,     // fewer matched features than min_corr: the outer iteration is skipped, the pose untouched
  kTermBarrierTimeout = 8, // k_linearize's grid barrier gave up
  kTermExchangeFailed = 9, // the peer-memory exchange of the rank sums failed
};

// ------------------------------------------------------------------------------------------------ Cholesky
// Two variants that round differently, so both stay: chol / chol_solve divide by the pivot (the odometry, the rig and logDet), chol6 /
// chol6_solve multiply by its reciprocal (the pose solve and the degeneracy test, whose single-thread step cannot afford a double division
// per entry).  In place, lower factor, row-major N x N; false when a pivot is not positive (the factor is then not usable).
template <int N>
__device__ __forceinline__ bool chol(double *A) {
  for (int j = 0; j < N; j++) {
    double d = A[j * N + j];
    for (int k = 0; k < j; k++) d -= A[j * N + k] * A[j * N + k];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    A[j * N + j] = d;
    for (int i = j + 1; i < N; i++) {
      double s = A[i * N + j];
      for (int k = 0; k < j; k++) s -= A[i * N + k] * A[j * N + k];
      A[i * N + j] = s / d;
    }
  }
  return true;
}
template <int N>
__device__ __forceinline__ void chol_solve(const double *L, const double *b, double *x) {
  double y[N];
#pragma unroll
  for (int i = 0; i < N; i++) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s -= L[i * N + k] * y[k];
    y[i] = s / L[i * N + i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {
    double s = y[i];
#pragma unroll
    for (int k = i + 1; k < N; k++) s -= L[k * N + i] * x[k];
    x[i] = s / L[i * N + i];
  }
}

// inv_diag[j] = 1 / L[j][j]: one square root and one division per column, the off-diagonal entries scaled by the reciprocal
__device__ __forceinline__ bool chol6(double *A, double *inv_diag) {
  constexpr int N = 6;
#pragma unroll
  for (int j = 0; j < N; j++) {
    double d = A[j * N + j];
#pragma unroll
    for (int k = 0; k < j; k++) d -= A[j * N + k] * A[j * N + k];
    if (!(d > 0.0)) return false;
    d = sqrt(d);
    A[j * N + j] = d;
    const double inv = 1.0 / d;
    inv_diag[j] = inv;
#pragma unroll
    for (int i = j + 1; i < N; i++) {
      double s = A[i * N + j];
#pragma unroll
      for (int k = 0; k < j; k++) s -= A[i * N + k] * A[j * N + k];
      A[i * N + j] = s * inv;
    }
  }
  return true;
}
__device__ __forceinline__ void chol6_solve(const double *L, const double *inv_diag, const double *b, double *x) {
  constexpr int N = 6;
  double y[6];
#pragma unroll
  for (int i = 0; i < N; i++) {
    double s = b[i];
#pragma unroll
    for (int k = 0; k < i; k++) s -= L[i * N + k] * y[k];
    y[i] = s * inv_diag[i];
  }
#pragma unroll
  for (int i = N - 1; i >= 0; i--) {
    double s = y[i];
#pragma unroll
    for (int k = i + 1; k < N; k++) s -= L[k * N + i] * x[k];
    x[i] = s * inv_diag[i];
  }
}

// ------------------------------------------------------------------------------------------------ the policy's rules
// LM diagonal entry of the Jacobi-scaled Hessian's diagonal entry h
__device__ __forceinline__ double lm_diag(double h) { return fmin(fmax(h, kMinDiag), kMaxDiag); }

// Verdict on the step to the candidate: a termination code (parameter tolerance, then function tolerance), or kLMAccept when the cost
// decreased by more than kMinRelDecrease of the model's prediction (rel: that ratio), or kLMReject.
enum LMVerdict : int { kLMAccept = -1, kLMReject = -2 };
__device__ __forceinline__ int lm_verdict(double step_norm, double x_norm, double cost, double new_cost, double model_cost_change, double &rel) {
  if (step_norm <= kParamTol * (x_norm + kParamTol)) return kTermParameterTol;
  const double cost_change = cost - new_cost;
  if (fabs(cost_change) <= kFuncTol * cost) return kTermFunctionTol;
  rel = cost_change / model_cost_change;
  return rel > kMinRelDecrease ? kLMAccept : kLMReject;
}

// Radius after an accepted step (the decrease factor goes back to kDecreaseFactor)
__device__ __forceinline__ double lm_radius_accept(double radius, double rel) {
  const double t = 2.0 * rel - 1.0;
  return fmin(kMaxRadius, radius / fmax(1.0 / 3.0, 1.0 - t * t * t));
}
// Radius and decrease factor after a rejected step
__device__ __forceinline__ void lm_radius_reject(double &radius, double &decrease_factor) {
  radius = radius / decrease_factor;
  decrease_factor = decrease_factor * 2.0;
}
// Radius after an invalid step (stop after kMaxInvalidSteps in a row)
__device__ __forceinline__ double lm_radius_invalid(double radius) { return radius * 0.5; }

// ------------------------------------------------------------------------------------------------ the single-thread machine
// A problem P supplies:
//   P::State              the state, with the fields x, xc (P::NX parameters in blocks of 7: accepted, candidate), H (D x D), g, cost,
//                         scale, diag, radius, decrease_factor, model_cost_change, x_norm, reuse_diagonal, iteration, num_invalid, done,
//                         termination, total_iterations, max_inner
//   P::D, P::NX           tangent and parameter dimensions
//   P::solve(A, b, x)     factor the damped system A in place and solve A x = b; false if A does not factor
//   P::plus(st, delta)    st->xc = st->x (+) delta
//   P::x_norm(st)         |x| over the free parameters
//   P::grad_max(st)       max |x - x (+) (-g)|, the gradient tolerance test's norm

// LevenbergMarquardtStrategy::ComputeStep and the invalid-step loop of TrustRegionMinimizer: returns with st->xc set, or with done.
template <class P>
__device__ void lm_compute_step(typename P::State *st) {
  constexpr int D = P::D;
  while (true) {
    if (st->iteration >= st->max_inner) {
      st->done = 1, st->termination = kTermMaxIterations;
      return;
    }
    double Hs[D * D], gs[D], A[D * D], step[D];
    for (int a = 0; a < D; a++) {
      gs[a] = st->scale[a] * st->g[a];
      for (int b = 0; b < D; b++) Hs[a * D + b] = st->scale[a] * st->H[a * D + b] * st->scale[b];
    }
    if (!st->reuse_diagonal)
      for (int j = 0; j < D; j++) st->diag[j] = lm_diag(Hs[j * D + j]);
    for (int i = 0; i < D * D; i++) A[i] = Hs[i];
    for (int j = 0; j < D; j++) {
      const double l = sqrt(st->diag[j] / st->radius);
      A[j * D + j] += l * l;
    }
    bool ok = P::solve(A, gs, step);
    if (ok)
      for (int j = 0; j < D; j++) {
        step[j] = -step[j];
        if (!isfinite(step[j])) ok = false;
      }
    st->reuse_diagonal = 1;
    st->iteration++;
    st->total_iterations++;
    double mcc = 0;
    if (ok) {
      double sg = 0, sHs = 0;
      for (int a = 0; a < D; a++) {
        sg += step[a] * gs[a];
        double t = 0;
        for (int b = 0; b < D; b++) t += Hs[a * D + b] * step[b];
        sHs += step[a] * t;
      }
      mcc = -(sg + 0.5 * sHs);
      if (mcc < 0) ok = false;
    }
    if (!ok) {
      if (++st->num_invalid >= kMaxInvalidSteps) {
        st->done = 1, st->termination = kTermInvalidSteps;
        return;
      }
      st->radius = lm_radius_invalid(st->radius);
      continue;
    }
    st->num_invalid = 0;
    double delta[D];
    for (int j = 0; j < D; j++) delta[j] = step[j] * st->scale[j];
    P::plus(st, delta);
    st->model_cost_change = mcc;
    return;
  }
}

// Mode 1: begin a solve; st->H, g and cost hold the evaluation at x.
template <class P>
__device__ void lm_begin(typename P::State *st) {
  st->x_norm = P::x_norm(st);
  for (int j = 0; j < P::D; j++) st->scale[j] = 1.0 / (1.0 + sqrt(st->H[j * P::D + j]));
  st->radius = kInitialRadius, st->decrease_factor = kDecreaseFactor, st->reuse_diagonal = 0;
  st->iteration = 0, st->num_invalid = 0, st->done = 0, st->termination = kTermMaxIterations;
  for (int k = 0; k < P::NX; k++) st->xc[k] = st->x[k];
  if (P::grad_max(st) <= kGradTol) {
    st->done = 1, st->termination = kTermGradientTol;
    return;
  }
  lm_compute_step<P>(st);
}

// Mode 2: digest the evaluation at the candidate (H, g, cost).  The step norm sums the blocks' squares parameter by parameter.
template <class P>
__device__ void lm_digest(typename P::State *st, const double *H, const double *g, double cost) {
  if (st->done) return;
  double sn = 0;
  for (int k = 0; k < 7; k++) {
    double t = 0;
    for (int b = k; b < P::NX; b += 7) t += (st->x[b] - st->xc[b]) * (st->x[b] - st->xc[b]);
    sn += t;
  }
  double rel;
  const int v = lm_verdict(sqrt(sn), st->x_norm, st->cost, cost, st->model_cost_change, rel);
  if (v >= 0) {
    st->done = 1, st->termination = v;
    return;
  }
  if (v == kLMAccept) {
    st->radius = lm_radius_accept(st->radius, rel);
    st->decrease_factor = kDecreaseFactor;
    st->reuse_diagonal = 0;
    for (int k = 0; k < P::NX; k++) st->x[k] = st->xc[k];
    st->x_norm = P::x_norm(st);
    for (int i = 0; i < P::D * P::D; i++) st->H[i] = H[i];
    for (int i = 0; i < P::D; i++) st->g[i] = g[i];
    st->cost = cost;
    if (P::grad_max(st) <= kGradTol) {
      st->done = 1, st->termination = kTermGradientTol;
      return;
    }
  } else {
    lm_radius_reject(st->radius, st->decrease_factor);
    st->reuse_diagonal = 1;
  }
  lm_compute_step<P>(st);
}

}  // namespace mloam
