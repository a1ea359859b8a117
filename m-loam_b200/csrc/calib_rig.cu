// calib_rig.cu — Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 over the whole rig (estimator.cpp:633-642, 670-787): one frame i,
// the reference LiDAR's LidarPureOdom* rows on pose_i (ext_ref constant, :642), every calibrated LiDAR n's LidarOnlineCalib* rows on ext_n
// (:714-735, :762-780), PriorFactor(tbl_[n], qbl_[n], PRIOR_FACTOR_POS, PRIOR_FACTOR_ROT) on every extrinsic when prior_factor is on
// (:675-685, prior_factor.hpp:27-72), one Levenberg-Marquardt over all blocks.
//
// The state is block-diagonal: block 0 is pose_i, block b >= 1 the extrinsic of the b-th calibrated LiDAR (index order, idx_ref
// skipped); no row couples two blocks.  Per outer iteration, whatever the rig size:
//   k_rig_poses      the pose each block's features are matched at (buildCalibMap, :1086-1090, :1135-1149)
//   k_rig_knn        one warp per feature of the whole rig: a segment table gives its LiDAR's block, map, n_neigh and pose; the
//                    search is the matcher's blind search (knn.cuh warp_knn, as k_match_knn runs it without a seed)
//   k_rig_fit        one thread per feature: match_fit.cuh fit_one with CHECK_FOV true
//   k_rig_linearize  one thread per feature: its 1x6 row on its block; per block 21 + 6 packed sums and a row count, plus the shared
//                    cost, reduced in a fixed order without atomics (as k_odom_linearize)
//   k_rig_lm         lm.cuh's state machine with one trust region over B blocks, on one warp: lane b scales, damps, factors and
//                    solves block b; step norm, x_norm and model cost change are summed across blocks in column order, so that a
//                    two-LiDAR rig without priors repeats the arithmetic of the coupled 12-dof [pose_i | ext_cal] solve bit for bit
// then max_inner x (k_rig_linearize + k_rig_lm) at the candidate.  mloam_calib_frame is the two-LiDAR case; with its communicator
// each evaluation adds k_rig_sum_partials and one all-reduce of B * 28 + 1 doubles before k_rig_lm.
#include <algorithm>
#include <climits>
#include <cmath>
#include <cstring>
#include <vector>

#include "ctx.h"
#include "factors.cuh"
#include "fit.cuh"
#include "host_util.h"
#include "knn.cuh"
#include "lm.cuh"
#include "match_fit.cuh"

namespace mloam {

constexpr int RIG_THREADS = 256;
constexpr int RIG_WARPS = RIG_THREADS / 32;
constexpr int RIG_L = MLOAM_MAX_LIDARS;
constexpr int RIG_SEGS = 2 * RIG_L;
constexpr int RIG_PB = 28;                       // per block: H upper (21) | g (6) | rows
constexpr int RIG_N = RIG_L * RIG_PB + 1;        // + the shared cost
constexpr int RIG_KMAX = 10;                     // neighbour slots per feature (n_neigh 5 uses the first 5)

// One segment: the corner or surf features of one LiDAR.  kind 1: the reference LiDAR (LidarPureOdom* on pose_i, n_neigh 5, the
// reference maps); kind 2: a calibrated LiDAR (LidarOnlineCalib* on its extrinsic, n_neigh 10, the calibration maps).
struct RigSeg {
  int off, n, map, blk, plane, kind;
};
struct RigSegs {
  RigSeg s[RIG_SEGS];
  MapView map[4];                // MLOAM_MAP_CORNER, MLOAM_MAP_SURF, then the calibrated LiDARs' corner / surf maps
  const float4 *pts;             // all features, segment after segment
  int *pos;                      // RIG_KMAX per feature
  unsigned char *valid;
  float *coeff;                  // 6 per feature
  int n_seg, n_total, B, sel_prune;
  float min_match_sq_dis, min_plane_dis;
  double huber_a;
};

struct RigState {
  double xp[7], xr[7];                           // pivot, ext_ref: constant
  double x[RIG_L][7], xc[RIG_L][7];              // accepted / candidate; block 0 pose_i, block b ext of a calibrated LiDAR
  double mpose[RIG_L][7];                        // match pose of each block
  double prior[RIG_L][7], prior_ref[7];          // PriorFactor targets of the blocks' extrinsics (block 0: unused) and of ext_ref
  double H[RIG_L][36], g[RIG_L][6], scale[RIG_L][6], diag[RIG_L][6];
  double Hs[RIG_L][36], A[RIG_L][36], gs[RIG_L][6], step[RIG_L][6];  // step scratch
  double cost, radius, decrease_factor, model_cost_change, x_norm, initial_cost, prior_pos, prior_rot;
  int B, has_prior, reuse_diagonal, iteration, num_invalid, done, termination, total_iterations, max_inner;
  int rows[RIG_L];                               // feature rows per block of the last evaluation
};

__constant__ double kRigI6[36] = {1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1};

__device__ __forceinline__ int rig_segment(const RigSegs &a, int i) {
  int s = 0;
  while (s + 1 < a.n_seg && i >= a.s[s + 1].off) s++;
  return s;
}

// ------------------------------------------------------------------------------------------ association
__global__ void k_rig_poses(RigState *st) {
  const int b = threadIdx.x;
  if (b >= st->B) return;
  double *o = st->mpose[b];
  if (b > 0) {
    for (int k = 0; k < 7; k++) o[k] = st->x[b][k];
    return;
  }
  // pivot^-1 * (pose_i * ext_ref)
  const PoseD P = pose_from_param(st->xp), I = pose_from_param(st->x[0]), R = pose_from_param(st->xr);
  const Q4 qpi = qconj(qnormalized(P.q));
  const Q4 q_ir = qmul(I.q, R.q);
  const D3 t_ir = qrot(I.q, R.t) + I.t;
  const Q4 q = qnormalized(qmul(qpi, q_ir));
  const D3 t = qrot(qpi, t_ir - P.t);
  o[0] = t.x, o[1] = t.y, o[2] = t.z, o[3] = q.x, o[4] = q.y, o[5] = q.z, o[6] = q.w;
}

template <int K>
__device__ __forceinline__ void rig_search(const MapView &map, const GridP &g, KnnSmem &ks, const float3 &sel, float min_match_sq_dis, int lane,
                                           int sel_prune, int *pos) {
  Best best;
  float explored = 0.0f;
  warp_knn<K, true, K + 1>(map, g, ks, sel.x, sel.y, sel.z, min_match_sq_dis, lane, best, &explored, 0.05f, nullptr, sel_prune != 0);
  const unsigned long long kK = best_key(best, K - 1);
  const bool ok = kK != MLOAM_KEY_NONE && key_d2(kK) < min_match_sq_dis;  // feature_extract.hpp:407,571,667,814
  if (lane < K) pos[lane] = ok ? best.pos : -1;
}

__global__ void __launch_bounds__(RIG_THREADS, 2) k_rig_knn(const __grid_constant__ RigSegs a, const RigState *st) {
  __shared__ KnnSmem ksm[RIG_WARPS];
  __shared__ GridP s_grid[4];
  __shared__ PoseD s_pose[RIG_L];
  const int lane = threadIdx.x & 31;
  KnnSmem &ks = ksm[threadIdx.x >> 5];
  knn_smem_init(ks, lane);
  if (threadIdx.x < 4) s_grid[threadIdx.x] = load_grid(a.map[threadIdx.x]);
  if (threadIdx.x < a.B) s_pose[threadIdx.x] = pose_from_param(st->mpose[threadIdx.x]);
  __syncthreads();
  for (int i = blockIdx.x * RIG_WARPS + (threadIdx.x >> 5); i < a.n_total; i += gridDim.x * RIG_WARPS) {
    const RigSeg &S = a.s[rig_segment(a, i)];
    const float4 p = __ldg(a.pts + i);
    const float3 sel = associate(s_pose[S.blk], p.x, p.y, p.z);  // pointAssociateToMap, utility.h:103-117
    int *pos = a.pos + (size_t)S.off * RIG_KMAX;
    if (S.kind == 1) rig_search<5>(a.map[S.map], s_grid[S.map], ks, sel, a.min_match_sq_dis, lane, a.sel_prune, pos + (size_t)(i - S.off) * 5);
    else rig_search<10>(a.map[S.map], s_grid[S.map], ks, sel, a.min_match_sq_dis, lane, a.sel_prune, pos + (size_t)(i - S.off) * 10);
  }
}

__global__ void __launch_bounds__(128) k_rig_fit(const __grid_constant__ RigSegs a, const RigState *st) {
  for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < a.n_total; i += gridDim.x * blockDim.x) {
    const RigSeg &S = a.s[rig_segment(a, i)];
    FitSet f;
    f.sorted = a.map[S.map].sorted, f.pts = a.pts + S.off, f.n = S.n, f.d_n = nullptr, f.pos = a.pos + (size_t)S.off * RIG_KMAX, f.half = 0;
    f.valid = a.valid + S.off, f.coeff = a.coeff + (size_t)S.off * 6, f.nn = nullptr, f.is_plane = S.plane, f.changed = nullptr;
    const PoseD T = pose_from_param(st->mpose[S.blk]);
    if (S.kind == 1) fit_one<5>(f, i - S.off, T, a.min_plane_dis, 1);
    else fit_one<10>(f, i - S.off, T, a.min_plane_dis, 1);
  }
}

// ------------------------------------------------------------------------------------------ linearisation
__global__ void __launch_bounds__(RIG_THREADS) k_rig_linearize(const __grid_constant__ RigSegs a, const RigState *st, int use_candidate, double *__restrict__ partials) {
  __shared__ double acc[RIG_WARPS][RIG_N];
  if (use_candidate && st->done) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int N = a.B * RIG_PB + 1;
  for (int k = lane; k < N; k += 32) acc[wid][k] = 0.0;
  __syncwarp();
  const double(*X)[7] = use_candidate ? st->xc : st->x;
  const Chain ch_ref = make_chain(st->xp, X[0], st->xr);
  for (int s = 0; s < a.n_seg; s++) {
    const RigSeg S = a.s[s];
    if (S.n <= 0) continue;
    const PoseR p_cal = make_poser(X[S.blk]);
    double *ac = acc[wid] + S.blk * RIG_PB;
    // all lanes of a warp iterate together (the shuffles below need them); out-of-range lanes contribute zeros
    for (int base = (blockIdx.x * RIG_WARPS + wid) * 32; base < S.n; base += gridDim.x * RIG_THREADS) {
      const int j = base + lane, i = S.off + j;
      double row[6];
#pragma unroll
      for (int k = 0; k < 6; k++) row[k] = 0.0;
      double r = 0.0, rho = 0.0, one = 0.0;
      if (j < S.n && a.valid[i]) {
        const float4 pf = __ldg(a.pts + i);
        const D3 p{(double)pf.x, (double)pf.y, (double)pf.z};
        const float *cf = a.coeff + (size_t)i * 6;
        const D3 c0{(double)cf[0], (double)cf[1], (double)cf[2]}, c1{(double)cf[3], (double)cf[4], (double)cf[5]};
        double J[6], Je[6];
        if (S.kind == 2) r = S.plane ? plane_factor(p_cal, p, c0, (double)cf[3], 1.0, J, true) : edge_factor(p_cal, p, c0, c1, 1.0, J, true);
        else if (S.plane) r = odom_plane_factor(ch_ref, p, c0, (double)cf[3], 1.0, nullptr, J, Je);
        else r = odom_edge_factor(ch_ref, p, c0, c1, 1.0, nullptr, J, Je);
        double rho1;
        huber(a.huber_a, r * r, &rho, &rho1);
        const double sc = sqrt(rho1);
        r = sc * r;
#pragma unroll
        for (int k = 0; k < 6; k++) row[k] = sc * J[k];
        one = 1.0;
      }
      int q = 0;
#pragma unroll
      for (int i0 = 0; i0 < 6; i0++) {
#pragma unroll
        for (int j0 = i0; j0 < 6; j0++) {
          double v = row[i0] * row[j0];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(MLOAM_FULL_MASK, v, o);
          if (lane == 0) ac[q] += v;
          q++;
        }
      }
#pragma unroll
      for (int k = 0; k < 8; k++) {
        double v = k < 6 ? row[k] * r : (k == 6 ? 0.5 * rho : one);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(MLOAM_FULL_MASK, v, o);
        if (lane == 0) {
          if (k < 6) ac[21 + k] += v;
          else if (k == 6) acc[wid][N - 1] += v;
          else ac[27] += v;
        }
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < N; k += RIG_THREADS) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < RIG_WARPS; w++) v += acc[w][k];
    partials[(size_t)blockIdx.x * N + k] = v;
  }
}

// ------------------------------------------------------------------------------------------ PriorFactor (prior_factor.hpp:36-71)
// residual = sqrt_info [P - pos_ ; 2 (rot_^-1 Q).vec],  sqrt_info = diag(pos_scale I3, rot_scale I3);
// jacobian (local, 6x6) = sqrt_info diag(I3, LeftQuatMatrix(Q^-1 rot_).topLeftCorner<3,3>()) — restated as written, including the
// rotation block the reference marks "seem to be wrong".  Eigen's inverse() is conjugate / squaredNorm.
__device__ __forceinline__ Q4 rig_qinv(const Q4 &q) {
  const double n2 = q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w;
  return {-q.x / n2, -q.y / n2, -q.z / n2, q.w / n2};
}
__device__ double rig_prior(const double *x, const double *x0, double sp, double sr, double *H36, double *g6) {
  const Q4 Q{x[3], x[4], x[5], x[6]}, R0{x0[3], x0[4], x0[5], x0[6]};
  const Q4 e = qmul(rig_qinv(R0), Q);
  double r[6] = {sp * (x[0] - x0[0]), sp * (x[1] - x0[1]), sp * (x[2] - x0[2]), sr * (2 * e.x), sr * (2 * e.y), sr * (2 * e.z)};
  if (H36) {
    const Q4 m = qmul(rig_qinv(Q), R0);
    // w I + [v]x
    const double L[9] = {m.w, -m.z, m.y, m.z, m.w, -m.x, -m.y, m.x, m.w};
    double J[36];
#pragma unroll
    for (int k = 0; k < 36; k++) J[k] = 0.0;
#pragma unroll
    for (int k = 0; k < 3; k++) J[k * 6 + k] = sp;
#pragma unroll
    for (int i = 0; i < 3; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) J[(3 + i) * 6 + 3 + j] = sr * L[i * 3 + j];
#pragma unroll
    for (int a = 0; a < 6; a++) {
      double s = 0;
#pragma unroll
      for (int i = 0; i < 6; i++) s += J[i * 6 + a] * r[i];
      g6[a] += s;
#pragma unroll
      for (int b = 0; b < 6; b++) {
        double h = 0;
#pragma unroll
        for (int i = 0; i < 6; i++) h += J[i * 6 + a] * J[i * 6 + b];
        H36[a * 6 + b] += h;
      }
    }
  }
  double c = 0;
#pragma unroll
  for (int i = 0; i < 6; i++) c += r[i] * r[i];
  return 0.5 * c;
}

// ------------------------------------------------------------------------------------------ LM over B blocks, one lane per block
// lane 0: sqrt of the sum of squares of the free blocks' parameters, block after block (od_xnorm's order)
__device__ double rig_xnorm(const RigState *st, const double (*x)[7]) {
  double s = 0;
  for (int b = 0; b < st->B; b++)
    for (int k = 0; k < 7; k++) s += x[b][k] * x[b][k];
  return sqrt(s);
}
// all lanes: max |x - x (+) (-g)| over the blocks
__device__ double rig_grad_max(const RigState *st, int lane) {
  double m = 0;
  if (lane < st->B) {
    double neg[6], xo[7];
    for (int j = 0; j < 6; j++) neg[j] = -st->g[lane][j];
    pose_plus(st->x[lane], neg, kRigI6, xo);
    for (int k = 0; k < 7; k++) m = fmax(m, fabs(st->x[lane][k] - xo[k]));
  }
  for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(MLOAM_FULL_MASK, m, o));
  return m;
}

// lm.cuh's lm_compute_step over the blocks: lane b owns block b; the decision is the warp's.  Returns with st->xc set, or with done.
__device__ void rig_compute_step(RigState *st, int lane) {
  const int B = st->B;
  while (true) {
    if (st->iteration >= st->max_inner) {
      __syncwarp();
      if (lane == 0) st->done = 1, st->termination = kTermMaxIterations;
      return;
    }
    bool ok = true;
    if (lane < B) {
      double *Hs = st->Hs[lane], *A = st->A[lane], *gs = st->gs[lane], *step = st->step[lane];
      const double *sc = st->scale[lane], *H = st->H[lane];
      for (int a = 0; a < 6; a++) {
        gs[a] = sc[a] * st->g[lane][a];
        for (int b = 0; b < 6; b++) Hs[a * 6 + b] = sc[a] * H[a * 6 + b] * sc[b];
      }
      if (!st->reuse_diagonal)
        for (int j = 0; j < 6; j++) st->diag[lane][j] = lm_diag(Hs[j * 6 + j]);
      for (int i = 0; i < 36; i++) A[i] = Hs[i];
      for (int j = 0; j < 6; j++) {
        const double l = sqrt(st->diag[lane][j] / st->radius);
        A[j * 6 + j] += l * l;
      }
      ok = chol<6>(A);
      if (ok) {
        chol_solve<6>(A, gs, step);
        for (int j = 0; j < 6; j++) {
          step[j] = -step[j];
          if (!isfinite(step[j])) ok = false;
        }
        // this block's columns of H s (the other blocks' columns are zero)
        for (int a = 0; a < 6; a++) {
          double t = 0;
          for (int b = 0; b < 6; b++) t += Hs[a * 6 + b] * step[b];
          A[a] = t;  // the factor is not needed any more
        }
      }
    }
    ok = __all_sync(MLOAM_FULL_MASK, ok);
    __syncwarp();
    double mcc = 0;
    if (lane == 0) {
      st->reuse_diagonal = 1;
      st->iteration++;
      st->total_iterations++;
      if (ok) {
        double sg = 0, sHs = 0;
        for (int b = 0; b < B; b++)
          for (int a = 0; a < 6; a++) {
            sg += st->step[b][a] * st->gs[b][a];
            sHs += st->step[b][a] * st->A[b][a];
          }
        mcc = -(sg + 0.5 * sHs);
      }
    }
    ok = __shfl_sync(MLOAM_FULL_MASK, ok && !(mcc < 0), 0);
    if (!ok) {
      int stop = 0;
      if (lane == 0) {
        if (++st->num_invalid >= kMaxInvalidSteps) st->done = 1, st->termination = kTermInvalidSteps, stop = 1;
        else st->radius = lm_radius_invalid(st->radius);
      }
      if (__shfl_sync(MLOAM_FULL_MASK, stop, 0)) return;
      __syncwarp();
      continue;
    }
    if (lane == 0) st->num_invalid = 0, st->model_cost_change = mcc;
    if (lane < B) {
      double delta[6];
      for (int j = 0; j < 6; j++) delta[j] = st->step[lane][j] * st->scale[lane][j];
      pose_plus(st->x[lane], delta, kRigI6, st->xc[lane]);
    }
    __syncwarp();
    return;
  }
}

// The feature sums of one evaluation (fixed-order sum over the CTAs' partials) into H / g of each block, with the blocks' priors at
// x; returns the cost (lane 0).
__device__ double rig_gather(RigState *st, const double *ne, const double (*x)[7], double (*H)[36], double (*g)[6], int lane) {
  const int B = st->B;
  double pc = 0.0;
  if (lane < B) {
    const double *e = ne + lane * RIG_PB;
    int q = 0;
    for (int i = 0; i < 6; i++)
      for (int j = i; j < 6; j++) H[lane][i * 6 + j] = H[lane][j * 6 + i] = e[q++];
    for (int k = 0; k < 6; k++) g[lane][k] = e[21 + k];
    if (st->has_prior && lane > 0) pc = rig_prior(x[lane], st->prior[lane], st->prior_pos, st->prior_rot, H[lane], g[lane]);
  }
  __syncwarp();
  double cost = ne[B * RIG_PB];
  for (int b = 1; b < B; b++) {
    const double v = __shfl_sync(MLOAM_FULL_MASK, pc, b);
    cost += v;
  }
  if (st->has_prior) cost += rig_prior(st->xr, st->prior_ref, st->prior_pos, st->prior_rot, nullptr, nullptr);  // constant ext_ref
  return cost;
}

// The N packed sums of one evaluation over the CTAs' partials, CTA after CTA
__device__ __forceinline__ void rig_sum_partials(const double *__restrict__ partials, int n_blocks, int N, double *ne) {
  for (int k = threadIdx.x; k < N; k += blockDim.x) {
    double v = 0.0;
    for (int b = 0; b < n_blocks; b++) v += partials[(size_t)b * N + k];
    ne[k] = v;
  }
}

// The sums a rank contributes to the all-reduce of a collective evaluation
__global__ void k_rig_sum_partials(const double *__restrict__ partials, int n_blocks, int N, double *__restrict__ ne) {
  rig_sum_partials(partials, n_blocks, N, ne);
}

__global__ void __launch_bounds__(RIG_THREADS) k_rig_lm(const double *__restrict__ partials, int n_blocks, RigState *st, int mode) {
  __shared__ double ne[RIG_N];
  __shared__ double cH[RIG_L][36], cg[RIG_L][6];
  const int B = st->B;
  rig_sum_partials(partials, n_blocks, B * RIG_PB + 1, ne);
  __syncthreads();
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  if (mode == 1) {
    const double cost = rig_gather(st, ne, st->x, st->H, st->g, lane);
    if (lane < B) {
      st->rows[lane] = (int)ne[lane * RIG_PB + 27];
      for (int j = 0; j < 6; j++) st->scale[lane][j] = 1.0 / (1.0 + sqrt(st->H[lane][j * 6 + j]));
      for (int k = 0; k < 7; k++) st->xc[lane][k] = st->x[lane][k];
    }
    if (lane == 0) {
      st->cost = st->initial_cost = cost;
      st->x_norm = rig_xnorm(st, st->x);
      st->radius = kInitialRadius, st->decrease_factor = kDecreaseFactor, st->reuse_diagonal = 0;
      st->iteration = 0, st->num_invalid = 0, st->done = 0, st->termination = kTermMaxIterations;
    }
    __syncwarp();
    if (rig_grad_max(st, lane) <= kGradTol) {
      if (lane == 0) st->done = 1, st->termination = kTermGradientTol;
      return;
    }
    rig_compute_step(st, lane);
    return;
  }
  if (st->done) return;
  const double cost = rig_gather(st, ne, st->xc, cH, cg, lane);
  int verdict = 0;  // lane 0's lm_verdict, broadcast below
  if (lane == 0) {
    double sn = 0;
    for (int k = 0; k < 7; k++) {
      double t = (st->x[0][k] - st->xc[0][k]) * (st->x[0][k] - st->xc[0][k]);
      for (int b = 1; b < B; b++) t += (st->x[b][k] - st->xc[b][k]) * (st->x[b][k] - st->xc[b][k]);
      sn += t;
    }
    sn = sqrt(sn);
    double rel;
    verdict = lm_verdict(sn, st->x_norm, st->cost, cost, st->model_cost_change, rel);
    if (verdict >= 0) {
      st->done = 1, st->termination = verdict;
    } else if (verdict == kLMAccept) {
      st->radius = lm_radius_accept(st->radius, rel);
      st->decrease_factor = kDecreaseFactor;
      st->reuse_diagonal = 0;
      st->cost = cost;
    } else {
      lm_radius_reject(st->radius, st->decrease_factor);
      st->reuse_diagonal = 1;
    }
  }
  verdict = __shfl_sync(MLOAM_FULL_MASK, verdict, 0);
  if (verdict >= 0) return;
  if (verdict == kLMAccept) {
    if (lane < B) {
      for (int k = 0; k < 7; k++) st->x[lane][k] = st->xc[lane][k];
      for (int i = 0; i < 36; i++) st->H[lane][i] = cH[lane][i];
      for (int i = 0; i < 6; i++) st->g[lane][i] = cg[lane][i];
    }
    __syncwarp();
    if (lane == 0) st->x_norm = rig_xnorm(st, st->x);
    __syncwarp();
    if (rig_grad_max(st, lane) <= kGradTol) {
      if (lane == 0) st->done = 1, st->termination = kTermGradientTol;
      return;
    }
  }
  __syncwarp();
  rig_compute_step(st, lane);
}

}  // namespace mloam

using namespace mloam;

static bool finite_n(const double *v, int n) {
  for (int k = 0; k < n; k++)
    if (!std::isfinite(v[k])) return false;
  return true;
}

// The rig problem after the callers' checks: per-LiDAR clouds and counts, the maps built.  prior7s nullable: no prior.  With a
// communicator (mloam_calib_frame's two ranks, each holding some LiDARs' features), every evaluation's packed sums and cost are
// all-reduced before the LM step, so that every rank takes the same step.
static int calib_rig_solve(Ctx *c, int n_lidars, int idx_ref, const mloam_point_t *const *surf, const int *surf_counts,
                           const mloam_point_t *const *corner, const int *corner_counts, const double *pose_pivot7, double *pose_i7,
                           double *ext7s, const double *prior7s, double prior_pos, double prior_rot, int max_outer, int max_inner,
                           double huber_a, int own_cal_maps, mloam_solve_stats_t *stats, int *h_rows) {
  const MapStorage *M = c->maps;
  const bool has_prior = prior7s != nullptr;
  long long n_surf = 0, n_corner = 0;
  for (int n = 0; n < n_lidars; n++) n_surf += surf_counts[n], n_corner += corner_counts[n];
  // blocks: 0 = pose_i (the reference LiDAR's rows), then the calibrated LiDARs in index order
  int blk_of[RIG_L], lidar_of[RIG_L];
  for (int n = 0, b = 1; n < n_lidars; n++) {
    const int bb = n == idx_ref ? 0 : b++;
    blk_of[n] = bb, lidar_of[bb] = n;
  }
  // segments: the reference LiDAR's corner and surf features, then each calibrated LiDAR's
  RigSegs sets;
  memset(&sets, 0, sizeof(sets));
  const int n_total = (int)(n_surf + n_corner);
  DevBuf &wb = c->rig_work;
  wb.in_graphs = false;  // no frame graph holds it
  int nb = 1;
  {
    int n_max = 1;
    for (int n = 0; n < n_lidars; n++) n_max = std::max(n_max, std::max(surf_counts[n], corner_counts[n]));
    nb = (n_max + RIG_THREADS - 1) / RIG_THREADS;
    nb = nb < 1 ? 1 : (nb > c->sm_count ? c->sm_count : nb);
  }
  float4 *d_pts;
  RigState *st;
  double *partials;
  MLOAM_CUDA_OK(c, carve(wb, [&](Carve &cv) {
    d_pts = cv.take<float4>((size_t)n_total + 1);
    sets.pos = cv.take<int>(RIG_KMAX * ((size_t)n_total + 1));
    sets.valid = cv.take<unsigned char>((size_t)n_total + 1);
    sets.coeff = cv.take<float>(6 * ((size_t)n_total + 1));
    st = cv.take<RigState>(1);
    partials = cv.take<double>((size_t)RIG_N * (nb + 1));  // + the all-reduced sums of a collective evaluation
  }));
  sets.pts = d_pts;
  int off = 0;
  for (int b = 0; b < n_lidars; b++) {
    const int n = lidar_of[b];
    for (int t = 0; t < 2; t++) {  // 0 corner, 1 surf
      RigSeg &S = sets.s[sets.n_seg++];
      S.off = off, S.n = t ? surf_counts[n] : corner_counts[n], S.blk = b, S.plane = t, S.kind = b == 0 ? 1 : 2;
      S.map = (b == 0 ? 0 : 2) + t;
      const mloam_point_t *src = t ? surf[n] : corner[n];
      if (S.n > 0) MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_pts + off, src, sizeof(float4) * (size_t)S.n, cudaMemcpyHostToDevice, c->stream));
      off += S.n;
    }
  }
  sets.map[0] = M[MLOAM_MAP_CORNER].view(), sets.map[1] = M[MLOAM_MAP_SURF].view();
  sets.map[2] = M[own_cal_maps ? MLOAM_MAP_SCAN_CORNER : MLOAM_MAP_CORNER].view();
  sets.map[3] = M[own_cal_maps ? MLOAM_MAP_SCAN_SURF : MLOAM_MAP_SURF].view();
  sets.n_total = n_total, sets.B = n_lidars, sets.sel_prune = c->knn_all_searches ? 0 : 1;
  sets.min_match_sq_dis = c->params.min_match_sq_dis, sets.min_plane_dis = c->params.min_plane_dis, sets.huber_a = huber_a;

  // the initial state goes up whole (the scratch and the LM fields are set by the first evaluation)
  std::vector<RigState> init(1);
  RigState &s0 = init[0];
  memset(&s0, 0, sizeof(s0));
  for (int k = 0; k < 7; k++) {
    s0.xp[k] = pose_pivot7[k], s0.xr[k] = ext7s[7 * idx_ref + k], s0.x[0][k] = pose_i7[k];
    for (int b = 1; b < n_lidars; b++) s0.x[b][k] = ext7s[7 * lidar_of[b] + k];
    if (has_prior) {
      s0.prior_ref[k] = prior7s[7 * idx_ref + k];
      for (int b = 1; b < n_lidars; b++) s0.prior[b][k] = prior7s[7 * lidar_of[b] + k];
    }
  }
  s0.prior_pos = prior_pos, s0.prior_rot = prior_rot, s0.has_prior = has_prior ? 1 : 0, s0.B = n_lidars, s0.max_inner = max_inner;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(st, &s0, sizeof(RigState), cudaMemcpyHostToDevice, c->stream));
  int *h_done = &c->pinned->done;
  int nbk = (n_total + RIG_WARPS - 1) / RIG_WARPS, nbf = (n_total + 127) / 128;
  nbk = nbk > 4 * c->sm_count ? 4 * c->sm_count : nbk;
  nbf = nbf > 4 * c->sm_count ? 4 * c->sm_count : nbf;
  const int N = n_lidars * RIG_PB + 1;
  // one LM evaluation: the per-feature sums at x (use_candidate 0) or at the candidate, then the LM step
  auto evaluate = [&](int use_candidate, int mode) -> int {
    k_rig_linearize<<<nb, RIG_THREADS, 0, c->stream>>>(sets, st, use_candidate, partials);
    c->launches += 2;
    if (!c->nccl_comm) {
      k_rig_lm<<<1, RIG_THREADS, 0, c->stream>>>(partials, nb, st, mode);
      return MLOAM_OK;
    }
    double *ne = partials + (size_t)RIG_N * nb;
    k_rig_sum_partials<<<1, 128, 0, c->stream>>>(partials, nb, N, ne);
    c->launches++;
    const int rc = comm_allreduce_doubles(c, ne, N);
    if (rc) return rc;
    k_rig_lm<<<1, RIG_THREADS, 0, c->stream>>>(ne, 1, st, mode);
    return MLOAM_OK;
  };
  for (int outer = 0; outer < max_outer; outer++) {
    k_rig_poses<<<1, 32, 0, c->stream>>>(st);
    c->launches++;
    if (n_total > 0) {
      k_rig_knn<<<nbk, RIG_THREADS, 0, c->stream>>>(sets, st);
      k_rig_fit<<<nbf, 128, 0, c->stream>>>(sets, st);
      c->launches += 2;
    }
    int rc = evaluate(0, 1);
    if (rc) return rc;
    for (int it = 0; it < max_inner; it++) {
      rc = evaluate(1, 2);
      if (rc) return rc;
      if (max_inner > 1) {
        MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_done, &st->done, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
        MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
        if (*h_done) break;
      }
    }
  }
  MLOAM_CUDA_OK(c, cudaGetLastError());
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(&s0, st, sizeof(RigState), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  for (int k = 0; k < 7; k++) {
    pose_i7[k] = s0.x[0][k];
    for (int b = 1; b < n_lidars; b++) ext7s[7 * lidar_of[b] + k] = s0.x[b][k];
  }
  int rows = 0;
  for (int b = 0; b < n_lidars; b++) rows += s0.rows[b];
  if (h_rows)
    for (int n = 0; n < n_lidars; n++) h_rows[n] = s0.rows[blk_of[n]];
  if (stats) {
    stats->ran = 1, stats->lm_iterations = s0.total_iterations, stats->termination = s0.termination, stats->final_cost = s0.cost;
    stats->n_surf = rows;  // feature rows of the last evaluation, all ranks
    stats->n_surf_in = (int)n_surf, stats->n_corner_in = (int)n_corner;
    for (int i = 0; i < 36; i++) stats->H[i] = s0.H[0][i];  // pose_i block
  }
  return MLOAM_OK;
}

// Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 for one frame i and the whole rig: see include/mloam_b200.h.
extern "C" int mloam_calib_rig(mloam_ctx_t *h, int n_lidars, int idx_ref, const mloam_point_t *h_surf, const int *surf_counts,
                               const mloam_point_t *h_corner, const int *corner_counts, const double *pose_pivot7, double *pose_i7,
                               double *ext7s, const double *prior7s, double prior_pos, double prior_rot, int max_outer, int max_inner,
                               double huber_a, int own_cal_maps, mloam_solve_stats_t *stats, int *h_rows) {
  if (!h) return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  if (n_lidars < 2 || n_lidars > RIG_L) return fail(c, MLOAM_E_INVALID, "calib_rig: n_lidars must be 2..16");
  if (idx_ref < 0 || idx_ref >= n_lidars) return fail(c, MLOAM_E_INVALID, "calib_rig: idx_ref outside 0..n_lidars-1");
  if (!surf_counts || !corner_counts || !pose_pivot7 || !pose_i7 || !ext7s) return fail(c, MLOAM_E_INVALID, "calib_rig: null counts or pose");
  if (max_outer < 1 || max_inner < 1) return fail(c, MLOAM_E_INVALID, "calib_rig: max_outer and max_inner must be >= 1");
  if (!std::isfinite(huber_a) || !std::isfinite(prior_pos) || !std::isfinite(prior_rot))
    return fail(c, MLOAM_E_INVALID, "calib_rig: non-finite huber_a or prior scale");
  if (!finite_n(pose_pivot7, 7) || !finite_n(pose_i7, 7) || !finite_n(ext7s, 7 * n_lidars))
    return fail(c, MLOAM_E_INVALID, "calib_rig: non-finite pivot, pose_i or extrinsic");
  const bool has_prior = prior_pos != 0.0 || prior_rot != 0.0;
  if (has_prior && (!prior7s || !finite_n(prior7s, 7 * n_lidars)))
    return fail(c, MLOAM_E_INVALID, "calib_rig: prior scales given without finite prior7s");
  long long n_surf = 0, n_corner = 0;
  for (int n = 0; n < n_lidars; n++) {
    if (surf_counts[n] < 0 || corner_counts[n] < 0) return fail(c, MLOAM_E_INVALID, "calib_rig: negative point count");
    n_surf += surf_counts[n], n_corner += corner_counts[n];
  }
  if ((n_surf > 0 && !h_surf) || (n_corner > 0 && !h_corner)) return fail(c, MLOAM_E_INVALID, "calib_rig: points counted without a cloud");
  if (n_surf + n_corner > INT_MAX / RIG_KMAX) return fail(c, MLOAM_E_INVALID, "calib_rig: too many features");
  cudaSetDevice(c->device);
  if (stats) memset(stats, 0, sizeof(*stats));
  if (multi_gpu(c)) return fail(c, MLOAM_E_STATE, "calib_rig: single-GPU; the two-rank calibration is mloam_calib_frame");
  const MapStorage *M = c->maps;
  if (!M[MLOAM_MAP_SURF].built || !M[MLOAM_MAP_CORNER].built) return fail(c, MLOAM_E_STATE, "calib_rig: build the local maps first");
  if (own_cal_maps && !(M[MLOAM_MAP_SCAN_SURF].built && M[MLOAM_MAP_SCAN_CORNER].built))
    return fail(c, MLOAM_E_STATE, "calib_rig: own_cal_maps needs MLOAM_MAP_SCAN_SURF / MLOAM_MAP_SCAN_CORNER built");
  const mloam_point_t *surf[RIG_L], *corner[RIG_L];
  long long so = 0, co = 0;
  for (int n = 0; n < n_lidars; n++) {
    surf[n] = h_surf ? h_surf + so : nullptr, corner[n] = h_corner ? h_corner + co : nullptr;
    so += surf_counts[n], co += corner_counts[n];
  }
  return calib_rig_solve(c, n_lidars, idx_ref, surf, surf_counts, corner, corner_counts, pose_pivot7, pose_i7, ext7s, has_prior ? prior7s : nullptr,
                         prior_pos, prior_rot, max_outer, max_inner, huber_a, own_cal_maps, stats, h_rows);
}

// Estimator::optimizeMap with ESTIMATE_EXTRINSIC == 1 for one frame i and one calibrated LiDAR: the rig problem of two LiDARs, the
// reference first (see include/mloam_b200.h).
extern "C" int mloam_calib_frame(mloam_ctx_t *h, const mloam_point_t *h_surf_ref, int n_surf_ref, const mloam_point_t *h_corner_ref,
                                 int n_corner_ref, const mloam_point_t *h_surf_cal, int n_surf_cal, const mloam_point_t *h_corner_cal,
                                 int n_corner_cal, const double *pose_pivot7, double *pose_i7, const double *ext_ref7, double *ext_cal7,
                                 int max_outer, int max_inner, double huber_a, int own_cal_maps, mloam_solve_stats_t *stats) {
  if (!h || !pose_pivot7 || !pose_i7 || !ext_ref7 || !ext_cal7 || n_surf_ref < 0 || n_corner_ref < 0 || n_surf_cal < 0 || n_corner_cal < 0 ||
      max_outer < 1 || max_inner < 1)
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (stats) memset(stats, 0, sizeof(*stats));
  const MapStorage *M = c->maps;
  if (!M[MLOAM_MAP_SURF].built || !M[MLOAM_MAP_CORNER].built) return fail(c, MLOAM_E_STATE, "calib_frame: build the local maps first");
  if (own_cal_maps && !(M[MLOAM_MAP_SCAN_SURF].built && M[MLOAM_MAP_SCAN_CORNER].built))
    return fail(c, MLOAM_E_STATE, "calib_frame: own_cal_maps needs MLOAM_MAP_SCAN_SURF / MLOAM_MAP_SCAN_CORNER built");
  const mloam_point_t *surf[2] = {h_surf_ref, h_surf_cal}, *corner[2] = {h_corner_ref, h_corner_cal};
  const int surf_counts[2] = {n_surf_ref, n_surf_cal}, corner_counts[2] = {n_corner_ref, n_corner_cal};
  for (int n = 0; n < 2; n++)
    if ((surf_counts[n] > 0 && !surf[n]) || (corner_counts[n] > 0 && !corner[n])) return MLOAM_E_INVALID;
  if ((long long)n_surf_ref + n_corner_ref + n_surf_cal + n_corner_cal > INT_MAX / RIG_KMAX) return MLOAM_E_INVALID;
  double ext7s[14];
  for (int k = 0; k < 7; k++) ext7s[k] = ext_ref7[k], ext7s[7 + k] = ext_cal7[k];
  const int rc = calib_rig_solve(c, 2, 0, surf, surf_counts, corner, corner_counts, pose_pivot7, pose_i7, ext7s, nullptr, 0.0, 0.0, max_outer,
                                 max_inner, huber_a, own_cal_maps, stats, nullptr);
  if (rc) return rc;
  for (int k = 0; k < 7; k++) ext_cal7[k] = ext7s[7 + k];
  return MLOAM_OK;
}
