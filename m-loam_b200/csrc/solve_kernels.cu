// solve_kernels.cu — residual/Jacobian evaluation, J^T J / J^T r reduction and the device-resident
// Levenberg-Marquardt state machine that replaces ceres::Solve for the single-pose problems of the path
// (lidar_mapper_keyframe.cpp:537-596, lidar_tracker.cpp:70-120).
//
//   k_linearize : one thread per feature -> (r, 1x6 row) in double, Huber corrector, per-thread packed
//                 upper-triangular J^T J (21) + J^T r (6) + cost + row counts, 31-exchange butterfly over the 30
//                 components -> shared-memory cross-warp sum -> one partial per block (deterministic: no atomics).
//                 The block that finishes last (ticket) runs lm_tail: fixed-order sum of the block partials, optional
//                 peer-memory exchange with the other GPUs' sums, and the LM state machine (Jacobi scaling, LM diagonal,
//                 6x6 Cholesky, step acceptance, radius update, tolerances, degeneracy remap) on a shared-memory copy of
//                 the device-resident state — the host only reads the final state back.
//   k_lm        : the same tail as a stand-alone kernel (NCCL path, mloam_normal_equations).
#include <cstddef>

#include "ctx.h"
#include "factors.cuh"
#include "lm.cuh"
#include "match_fit.cuh"

namespace mloam {

constexpr int NE_H = 21, NE_G = 6;
constexpr int NE_PACK = 30;  // 21 H upper | 6 g | cost | rows(set 0) | rows(set 1)
constexpr int LIN_THREADS = 256;
constexpr int LM_THREADS = 256;

struct FeatSetDev {
  const float4 *pts;
  const unsigned char *valid;
  const float *coeff;
  int n;
  int is_plane;
  const int *d_n;
  const double *sinfo;
  const unsigned char *mask;
};
struct LinArgs {
  FeatSetDev set[2];
  int n_sets;
  double sqrt_info, huber_a;
  const double *pose;      // explicit pose (7 doubles) or null
  const LMState *state;    // state->x (use_state 1) / state->xc (use_state 2)
  int use_state;
  int respect_done;
  // fused LM tail (single GPU): the block that finishes last reduces the partials and advances the state machine
  int lm_mode;             // 1 | 2, or 0: no tail (partials only)
  int lm_serial;           // the tail's state machine on one thread (MLOAM_LM_TAIL=serial) instead of one warp
  int want_eig;
  double eig_thre;
  unsigned *ticket;        // zero between launches
  LMState *state_rw;
  const P2PView *p2p;      // device copy of the peer-memory view, or null: sum the packed normal equations over the ranks
  // two_pass (needs the fused tail): the evaluation at x, the LM step, and the evaluation at the candidate xc in ONE launch.  The
  // blocks wait at a grid barrier (generation word next to the ticket) for the block that ran the tail; every block of the grid
  // is resident (<= 64 blocks of 256 threads, one per SM).
  int two_pass;
  // deferred fit (KFIT > 0): the thread that evaluates a feature first fits its line / plane from the matcher's neighbour list
  FitSet fit[2];
  float fit_min_plane_dis;
  int fit_check_fov;
  // speculative schedule (SpecState, with the deferred fit): fit from the lists matched at spec->xc only when x is that pose,
  // commit the choice in the tail and, with spec_publish, hand the new candidate to the next matcher
  SpecState *spec;
  int spec_publish;
  // MLOAM_LIN_TRACE=1 only (the k_linearize<KFIT, true> instance): LIN_TRACE_BLOCK words per block of pass 0's phase stamps
  unsigned long long *trace;
};

// Phase stamps of pass 0 (diagnosis).  Per block: for warp w, words 4w..4w+3 = [%globaltimer at entry (lane 0), ns from there to
// the end of the feature loop (slowest lane), fit cycles (slowest lane, clock64), feature-loop cycles (slowest lane)]; then words
// 32..35 = %globaltimer of thread 0 after the block partial is written, after the ticket, and (last block only) at the tail's
// start and end.
constexpr int LIN_TRACE_BLOCK = 64;
constexpr int LIN_TRACE_SLOT = 64 * LIN_TRACE_BLOCK;  // <= 64 blocks
constexpr int LIN_TRACE_SLOTS = 16;

__device__ __forceinline__ unsigned long long global_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
  return t;
}

// Loss-corrected row of one point-to-plane / point-to-line feature at pose P: returns r and scales J by sqrt(rho'(r^2)); *rho = Huber(r^2).
// cf: the feature's 6 coefficients (fs.coeff + 6 i, or the fit just computed).
__device__ __forceinline__ double map_factor_row(const PoseR &P, const FeatSetDev &fs, int i, const float (&cf)[6], double sqrt_info,
                                                 double huber_a, double *J, double *rho) {
  const float4 pf = __ldg(fs.pts + i);
  const D3 p{(double)pf.x, (double)pf.y, (double)pf.z};
  const double si = fs.sinfo ? fs.sinfo[i] : sqrt_info;  // per-feature weight when mapping is uncertainty-aware
  double r;
  if (fs.is_plane) {
    r = plane_factor(P, p, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, (double)cf[3], si, J, true);
  } else {
    r = edge_factor(P, p, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, D3{(double)cf[3], (double)cf[4], (double)cf[5]}, si, J, true);
  }
  double rho1;
  huber(huber_a, r * r, rho, &rho1);
  const double sc = sqrt(rho1);
#pragma unroll
  for (int k = 0; k < 6; k++) J[k] = sc * J[k];
  return sc * r;
}
__device__ __forceinline__ double map_factor_row(const PoseR &P, const FeatSetDev &fs, int i, double sqrt_info, double huber_a, double *J,
                                                 double *rho) {
  float cf[6];
#pragma unroll
  for (int k = 0; k < 6; k++) cf[k] = fs.coeff[(size_t)i * 6 + k];
  return map_factor_row(P, fs, i, cf, sqrt_info, huber_a, J, rho);
}

template <bool SERIAL>
__device__ __noinline__ void lm_tail(const double *partials, int n_blocks, LMState *gst, int mode, double eig_thre, int want_eig, double *out_ne,
                                     const P2PView *p2p, double *xc_pub);

// One offset of k_linearize's warp butterfly.  O is a template argument so that every index of v is a constant: with a loop over
// the offsets the compiler kept v in local memory (a 256 B store and dependent reloads per thread on the way to the block partial).
template <int O>
__device__ __forceinline__ void butterfly_stage(double (&v)[32], int lane) {
  const bool upper = (lane & O) != 0;
#pragma unroll
  for (int k = 0; k < O; k++) {
    const double send = upper ? v[k] : v[k + O];
    const double keep = upper ? v[k + O] : v[k];
    v[k] = keep + __shfl_xor_sync(MLOAM_FULL_MASK, send, O);
  }
}

template <int KFIT, bool TRACE = false>
__global__ void __launch_bounds__(LIN_THREADS) k_linearize(LinArgs a, double *__restrict__ partials) {
  __shared__ double sm[LIN_THREADS / 32][NE_PACK];
  __shared__ bool is_last;
  __shared__ int barrier_failed;
  unsigned long long *const tr = TRACE ? a.trace + (size_t)blockIdx.x * LIN_TRACE_BLOCK : nullptr;
  // Programmatic dependent launch: everything below reads what the previous kernel of the GN chain writes (state->done / x, the
  // SpecState, the matcher's lists for the fit, the ticket and generation word k_eval_candidate shares), so the wait comes first
  cudaGridDependencySynchronize();
  cudaTriggerProgrammaticLaunchCompletion();
  unsigned long long t_entry = 0ull;
  long long c_entry = 0ll, c_fit = 0ll;
  if (TRACE) t_entry = global_ns(), c_entry = clock64();
  if (a.respect_done && a.state && a.state->done) {  // Solve already terminated: nothing to evaluate
    if (a.lm_mode != 0 && blockIdx.x == 0 && threadIdx.x == 0) a.state_rw->work[0] = 0, a.state_rw->work[1] = 0;
    return;
  }
  volatile unsigned *const gen = a.ticket + 1;
  const unsigned gen0 = a.two_pass ? *gen : 0u;  // read before this block's ticket: the release cannot have happened yet
  // speculative schedule: the lists the last matcher wrote (half sel ^ 1) were matched at spec->xc; they are the lists at x iff
  // x is that pose bit for bit (the step was taken).  Otherwise x did not move and the lists, valid and coeff of half sel stand.
  // Every load here is independent of the others (no short-circuit between them), so they are in flight together.
  int spec_sel = 0;
  bool spec_hit = true;
  if (a.spec) {
    spec_sel = a.spec->sel & 1;  // read as k_match_knn reads it
#pragma unroll
    for (int k = 0; k < 7; k++) spec_hit = spec_hit & (__double_as_longlong(a.state->x[k]) == __double_as_longlong(a.spec->xc[k]));
  }
  // the device-side feature counts are written before the launch and read by both passes
  int set_n[2];
#pragma unroll
  for (int s = 0; s < 2; s++) set_n[s] = s < a.n_sets ? (a.set[s].d_n ? min(a.set[s].n, *a.set[s].d_n) : a.set[s].n) : 0;
#pragma unroll 1
  for (int pass = 0; pass < (a.two_pass ? 2 : 1); pass++) {
  double xs[7];
  if (pass == 0) {
    const double *px = a.use_state == 1 ? a.state->x : (a.use_state == 2 ? a.state->xc : a.pose);
#pragma unroll
    for (int k = 0; k < 7; k++) xs[k] = px[k];
  } else {
    // grid barrier: the block that ran the tail of pass 0 publishes the state and bumps the generation word
    if (threadIdx.x == 0) {
      barrier_failed = 0;
      const long long w0 = clock64();
      while (*gen == gen0) {
        if (clock64() - w0 > 4000000000ll) {  // ~2 s: a block of this grid never became resident
          barrier_failed = 1;
          break;
        }
      }
      __threadfence();
    }
    __syncthreads();
    if (barrier_failed) {
      if (threadIdx.x == 0) a.state_rw->termination = kTermBarrierTimeout, a.state_rw->done = 1;
      return;
    }
    if (__ldcg(&a.state_rw->done)) return;  // the step of pass 0 ended the Solve (tolerance, too few rows, invalid steps)
#pragma unroll
    for (int k = 0; k < 7; k++) xs[k] = __ldcg(&a.state_rw->xc[k]);  // L2: this SM's L1 may hold the line from pass 0
  }
  const PoseR P = make_poser(xs);
  double acc[NE_PACK];
#pragma unroll
  for (int k = 0; k < NE_PACK; k++) acc[k] = 0.0;
  for (int s = 0; s < a.n_sets; s++) {
    const FeatSetDev fs = a.set[s];
    const int fn = set_n[s & 1];
    // Both sets keep their features at the low indices of a much larger launch bound: the second set is handed out from
    // the last thread downwards, so that a thread evaluates one feature of either set instead of one of each.
    const int G = gridDim.x * blockDim.x, gid = blockIdx.x * blockDim.x + threadIdx.x;
    for (int i = (s & 1) ? G - 1 - gid : gid; i < fn; i += G) {
      // valid as it stands, read before the fit so that the two loads overlap; a fit replaces it (and coeff) from registers
      bool valid = fs.valid[i] != 0, fitted = false;
      float fit_c[6];
      if (KFIT > 0 && pass == 0 && a.fit[s].pos && spec_hit) {  // deferred fit: this thread is the only one that touches feature i
        constexpr int KF = KFIT > 0 ? KFIT : 5;
        const PoseD T = pose_from_param(xs);
        FitSet f = a.fit[s];
        f.pos += (size_t)(spec_sel ^ 1) * f.half * KF;  // half 0 when the lists are not double-buffered (f.half == 0)
        const long long c0 = TRACE ? clock64() : 0ll;
        bool fit_ok = false;
        fitted = fit_one<KF>(f, i, T, a.fit_min_plane_dis, a.fit_check_fov, &fit_ok, fit_c);
        if (fitted) valid = fit_ok;
        if (TRACE) c_fit += clock64() - c0;
      }
      if (!valid || (fs.mask && !fs.mask[i])) continue;
      if (fs.is_plane == 2) {
        const float4 pf = __ldg(fs.pts + i);
        const D3 p{(double)pf.x, (double)pf.y, (double)pf.z};
        const float *cf = fs.coeff + (size_t)i * 6;
        // LidarScanEdgeFactorVector (tracker, lidar_tracker.cpp:89): one 3-row residual BLOCK, the loss acts on
        // its squared norm (Ceres applies rho per block)
        double r3[3], J3[18];
        edge_vector_factor(P, p, D3{(double)cf[0], (double)cf[1], (double)cf[2]}, D3{(double)cf[3], (double)cf[4], (double)cf[5]}, r3,
                           J3, true);
        double rho, rho1;
        huber(a.huber_a, r3[0] * r3[0] + r3[1] * r3[1] + r3[2] * r3[2], &rho, &rho1);
        const double sc = sqrt(rho1);
#pragma unroll
        for (int m = 0; m < 3; m++) {
          const double rm = sc * r3[m];
          double Jm[6];
#pragma unroll
          for (int k = 0; k < 6; k++) Jm[k] = sc * J3[m * 6 + k];
          int q = 0;
#pragma unroll
          for (int i0 = 0; i0 < 6; i0++)
#pragma unroll
            for (int j0 = i0; j0 < 6; j0++) acc[q++] += Jm[i0] * Jm[j0];
#pragma unroll
          for (int k = 0; k < 6; k++) acc[NE_H + k] += Jm[k] * rm;
        }
        acc[NE_H + NE_G] += 0.5 * rho;
        if (s == 0) acc[NE_H + NE_G + 1] += 1.0;
        else acc[NE_H + NE_G + 2] += 1.0;
        continue;
      }
      float cf[6];
#pragma unroll
      for (int k = 0; k < 6; k++) cf[k] = fitted ? fit_c[k] : fs.coeff[(size_t)i * 6 + k];
      double J[6], rho;
      const double r = map_factor_row(P, fs, i, cf, a.sqrt_info, a.huber_a, J, &rho);
      int q = 0;
#pragma unroll
      for (int i0 = 0; i0 < 6; i0++)
#pragma unroll
        for (int j0 = i0; j0 < 6; j0++) acc[q++] += J[i0] * J[j0];
#pragma unroll
      for (int k = 0; k < 6; k++) acc[NE_H + k] += J[k] * r;
      acc[NE_H + NE_G] += 0.5 * rho;
      if (s == 0) acc[NE_H + NE_G + 1] += 1.0;
      else acc[NE_H + NE_G + 2] += 1.0;
    }
  }
  // Warp reduction of all 30 components at once (fixed butterfly, 31 exchanges instead of 30 x 5): at offset o a lane
  // keeps the half of its remaining components selected by its bit o and adds the partner's partial sums of that
  // half; after offsets 16..1 lane L holds the warp total of component L.
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (TRACE && pass == 0) {
    const unsigned long long t0 = __shfl_sync(MLOAM_FULL_MASK, t_entry, 0);
    const unsigned loop_ns = __reduce_max_sync(MLOAM_FULL_MASK, (unsigned)(global_ns() - t0));
    const unsigned loop_cyc = __reduce_max_sync(MLOAM_FULL_MASK, (unsigned)(clock64() - c_entry));
    const unsigned fit_cyc = __reduce_max_sync(MLOAM_FULL_MASK, (unsigned)c_fit);
    if (lane == 0) tr[4 * wid] = t0, tr[4 * wid + 1] = loop_ns, tr[4 * wid + 2] = fit_cyc, tr[4 * wid + 3] = loop_cyc;
  }
  {
    double v[32];
#pragma unroll
    for (int k = 0; k < 32; k++) v[k] = k < NE_PACK ? acc[k] : 0.0;
    butterfly_stage<16>(v, lane);
    butterfly_stage<8>(v, lane);
    butterfly_stage<4>(v, lane);
    butterfly_stage<2>(v, lane);
    butterfly_stage<1>(v, lane);
    if (lane < NE_PACK) sm[wid][lane] = v[0];
  }
  __syncthreads();
  if (threadIdx.x < NE_PACK) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < LIN_THREADS / 32; w++) v += sm[w][threadIdx.x];
    partials[(size_t)blockIdx.x * NE_PACK + threadIdx.x] = v;
    if (TRACE && pass == 0 && threadIdx.x == 0) tr[32] = global_ns();
  }
  if (a.lm_mode == 0) return;
  // ---- fused tail: the last block to arrive sums the partials in block order (so the result does not depend on
  // which block that is) and runs the LM step that a separate k_lm launch used to do.
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (TRACE && pass == 0 && threadIdx.x == 0) tr[33] = global_ns(), tr[34] = 0ull, tr[35] = 0ull;
  if (!is_last) {
    if (a.two_pass && pass == 0) continue;  // on to the barrier of pass 1
    return;
  }
  __threadfence();
  // with spec_publish the tail also copies the new candidate to where the next matcher searches (every block has read the old one)
  {
    const int mode = pass == 0 ? a.lm_mode : 2, want_eig = pass == 0 ? a.want_eig : 1;
    double *const xc_pub = (a.spec && a.spec_publish && pass == 0) ? a.spec->xc : nullptr;
    if (TRACE && pass == 0 && threadIdx.x == 0) tr[34] = global_ns();
    if (a.lm_serial) lm_tail<true>(partials, (int)gridDim.x, a.state_rw, mode, a.eig_thre, want_eig, nullptr, a.p2p, xc_pub);
    else lm_tail<false>(partials, (int)gridDim.x, a.state_rw, mode, a.eig_thre, want_eig, nullptr, a.p2p, xc_pub);
  }
  __threadfence();  // the state (written by all threads of this block) before the ticket reset and the release
  __syncthreads();
  if (TRACE && pass == 0 && threadIdx.x == 0) tr[35] = global_ns();
  if (threadIdx.x == 0) {
    if (a.spec && pass == 0 && spec_hit) a.spec->sel = spec_sel ^ 1;  // every block has read sel and fitted: commit
    *a.ticket = 0u;
    if (a.two_pass && pass == 0) {
      __threadfence();
      atomicAdd(a.ticket + 1, 1u);  // release the grid into pass 1
    }
  }
  }
}

// ---------------------------------------------------------------------------------------- small dense (device)
__host__ __device__ void eig_sym6(const double *Ain, double *w, double *V) {
  const int N = 6;
  double a[36], v[36];
  for (int i = 0; i < 36; i++) a[i] = Ain[i], v[i] = (i % 7 == 0) ? 1.0 : 0.0;
  for (int sweep = 0; sweep < 60; sweep++) {
    double off = 0, diag = 0;
    for (int i = 0; i < N; i++) {
      diag += fabs(a[i * N + i]);
      for (int j = i + 1; j < N; j++) off += fabs(a[i * N + j]);
    }
    if (off <= 1e-22 * diag || off == 0.0) break;
    for (int p = 0; p < N - 1; p++)
      for (int q = p + 1; q < N; q++) {
        const double apq = a[p * N + q];
        if (apq == 0.0) continue;
        const double theta = (a[q * N + q] - a[p * N + p]) / (2.0 * apq);
        double t = 1.0 / (fabs(theta) + sqrt(theta * theta + 1.0));
        if (theta < 0.0) t = -t;
        const double c = 1.0 / sqrt(t * t + 1.0), s = t * c;
        a[p * N + p] -= t * apq;
        a[q * N + q] += t * apq;
        a[p * N + q] = a[q * N + p] = 0.0;
        for (int r = 0; r < N; r++) {
          if (r == p || r == q) continue;
          const double arp = a[r * N + p], arq = a[r * N + q];
          a[r * N + p] = a[p * N + r] = c * arp - s * arq;
          a[r * N + q] = a[q * N + r] = s * arp + c * arq;
        }
        for (int k = 0; k < N; k++) {
          const double vkp = v[k * N + p], vkq = v[k * N + q];
          v[k * N + p] = c * vkp - s * vkq;
          v[k * N + q] = s * vkp + c * vkq;
        }
      }
  }
  int idx[6] = {0, 1, 2, 3, 4, 5};
  for (int i = 1; i < N; i++) {  // stable insertion sort, ascending
    int k = idx[i], j = i - 1;
    while (j >= 0 && a[idx[j] * N + idx[j]] > a[k * N + k]) idx[j + 1] = idx[j], j--;
    idx[j + 1] = k;
  }
  for (int j = 0; j < N; j++) {
    w[j] = a[idx[j] * N + idx[j]];
    for (int k = 0; k < N; k++) V[k * N + j] = v[k * N + idx[j]];
  }
}

// Eigenvalue report of a non-degenerate Solve, filled in by the host from the read-back H0 (the device only runs the
// 6x6 Jacobi solver when the Cholesky test says a direction is degenerate — a ~10^5-cycle single-thread job).
void eig_report_host(const double *H36, double *w6) {
  double V[36];
  eig_sym6(H36, w6, V);
}

// The pose problem of the single-thread machine (lm.cuh): one 6-DoF block, x (+) delta through the degeneracy remap V_update, chol6.
struct PoseProblem {
  using State = LMState;
  static constexpr int D = 6, NX = 7;
  __device__ static bool solve(double *A, const double *b, double *x) {
    double inv_diag[6];
    if (!chol6(A, inv_diag)) return false;
    chol6_solve(A, inv_diag, b, x);
    return true;
  }
  __device__ static void plus(LMState *st, const double *delta) { pose_plus(st->x, delta, st->V_update, st->xc); }
  __device__ static double x_norm(const LMState *st) {
    double xn = 0;
    for (int k = 0; k < 7; k++) xn += st->x[k] * st->x[k];
    return sqrt(xn);
  }
  __device__ static double grad_max(const LMState *st) {
    double neg[6], xp[7];
    for (int j = 0; j < 6; j++) neg[j] = -st->g[j];
    pose_plus(st->x, neg, st->V_update, xp);
    double m = 0;
    for (int k = 0; k < 7; k++) m = fmax(m, fabs(st->x[k] - xp[k]));
    return m;
  }
};

__device__ void unpack_ne(const double *ne, double *H, double *g) {
  int q = 0;
  for (int i = 0; i < 6; i++)
    for (int j = i; j < 6; j++) {
      H[i * 6 + j] = ne[q];
      H[j * 6 + i] = ne[q];
      q++;
    }
  for (int k = 0; k < 6; k++) g[k] = ne[NE_H + k];
}

// evalDegenracy's eigen-decomposition of st->H and the remapped V_update (PoseLocalParameterization::setParameter) of a (nearly)
// degenerate Solve; one thread.
__device__ void eig_remap(LMState *st, double eig_thre) {
  double w[6], Vf[36], Vp[36];
  eig_sym6(st->H, w, Vf);
  for (int i = 0; i < 36; i++) Vp[i] = Vf[i];
  for (int j = 0; j < 6; j++) {
    if (w[j] < eig_thre) {
      for (int k = 0; k < 6; k++) Vp[k * 6 + j] = 0.0;
      st->is_degenerate = 1;
    } else {
      break;
    }
  }
  for (int i = 0; i < 6; i++) st->eig[i] = w[i];
  if (st->is_degenerate)
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) {
        double s = 0;
        for (int k = 0; k < 6; k++) s += Vf[i * 6 + k] * Vp[j * 6 + k];
        st->V_update[i * 6 + j] = s;
      }
}

// One thread advances the state machine on a shared-memory copy of the state (lm_tail stages it in and out): the pose's prologue of
// a Solve around lm.cuh's machine.  mode 1: begin a Solve with the evaluation at x.  mode 2: digest the evaluation at xc.
// The reference for lm_advance_warp (MLOAM_LM_TAIL=serial).
__device__ void lm_advance(LMState *st, const double *ne, int mode, double eig_thre, int want_eig) {
  double H[36], g[6];
  unpack_ne(ne, H, g);
  const double cost = ne[NE_H + NE_G];
  if (mode == 2) {
    lm_digest<PoseProblem>(st, H, g, cost);
    return;
  }
  for (int i = 0; i < 36; i++) st->H[i] = H[i], st->H0[i] = H[i];
  for (int i = 0; i < 6; i++) st->g[i] = g[i];
  st->cost = cost;
  st->initial_cost = cost;
  st->n_valid[0] = (int)ne[NE_H + NE_G + 1];
  st->n_valid[1] = (int)ne[NE_H + NE_G + 2];
  st->rows = st->n_valid[0] + st->n_valid[1];
  st->skipped = 0;
  if (st->rows < st->min_corr) {  // "less correspondence": the outer iteration is skipped, pose untouched
    st->done = 1, st->termination = kTermTooFewRows, st->skipped = 1;
    for (int k = 0; k < 7; k++) st->xc[k] = st->x[k];
    return;
  }
  // PoseLocalParameterization::setParameter + evalDegenracy (lidar_mapper_keyframe.cpp:1172-1204)
  for (int i = 0; i < 36; i++) st->V_update[i] = (i % 7 == 0) ? 1.0 : 0.0;
  st->is_degenerate = 0;
  for (int i = 0; i < 6; i++) st->eig[i] = 0.0;
  // lambda_min(H) > eig_thre  <=>  H - eig_thre*I is positive definite: one 6x6 Cholesky decides the common,
  // non-degenerate case; the Jacobi eigen-solver only runs when a direction is (nearly) degenerate or when the
  // caller asked for the eigenvalue report (want_eig: last outer iteration).
  bool need_eig = st->rows > 0 && eig_thre > 0.0;
  if (need_eig && !want_eig) {
    double S[36];
    for (int i = 0; i < 36; i++) S[i] = H[i] - ((i % 7 == 0) ? eig_thre : 0.0);
    double inv_diag[6];
    if (chol6(S, inv_diag)) need_eig = false;
  }
  if (need_eig) eig_remap(st, eig_thre);
  lm_begin<PoseProblem>(st);
}

// ---------------------------------------------------------------------------------------- the LM step on one warp
// lm_advance on the 32 lanes of warp 0 of the tail block, with the serial code's operations in its order (everything is compiled
// -fmad=false, so the state is bit-identical).  A 6x6 is held by rows: lane 8 q + i owns row i of group q's matrix (rows 6 and 7 of a
// group are padding), so group 0 factors the damped LM system while group 1 factors H - eig_thre I for the degeneracy test, in one
// instruction stream; each column's pivot row is broadcast by shuffle.  The Jacobi scaling takes one lane per column, the gradient
// test and the candidate pose run their pose_plus side by side on lanes 0 and 1, and scalars are computed redundantly by every lane
// (no divergence, no broadcast).  Only lane 0 writes scalar fields of the shared state; __syncwarp orders reads, writes and re-reads.

// chol6 by rows: lane (lane & ~7) + i holds row i in a[]; inv_diag[j] = 1 / L[j][j] of the lane's group.  Returns chol6's verdict
// for the lane's group; after a failed pivot the group computes on with NaNs and the factor is not used.
__device__ __forceinline__ bool chol6_rows(double a[6], double inv_diag[6]) {
  const int lane = threadIdx.x & 31, base = lane & ~7, r = lane & 7;
  bool ok = true;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    double d = a[j];
#pragma unroll
    for (int k = 0; k < j; k++) d -= a[k] * a[k];
    d = __shfl_sync(MLOAM_FULL_MASK, d, base + j);
    ok = ok && d > 0.0;
    d = sqrt(d);
    const double inv = 1.0 / d;
    inv_diag[j] = inv;
    double pj[6];
#pragma unroll
    for (int k = 0; k < j; k++) pj[k] = __shfl_sync(MLOAM_FULL_MASK, a[k], base + j);
    if (r == j) a[j] = d;
    if (r > j) {
      double s = a[j];
#pragma unroll
      for (int k = 0; k < j; k++) s -= a[k] * pj[k];
      a[j] = s * inv;
    }
  }
  return ok;
}

struct StepTry {
  bool ok;          // lm_compute_step's ok: the damped system factored, the step is finite and the model cost decreases
  bool deg_ok;      // with the degeneracy test: H - eig_thre I is positive definite
  double mcc;       // model cost change
  double step[6];   // scaled step
  double diag[6];   // LM diagonal the step used
};

// The arithmetic of one pass of lm_compute_step's loop (not its bookkeeping) on the state st: group 0 solves the damped scaled
// system, group 1 factors H - eig_thre I (read with deg_test).  Every lane returns the same values.
__device__ __forceinline__ StepTry lm_try_step_warp(const LMState *st, bool deg_test, double eig_thre) {
  const int lane = threadIdx.x & 31, grp = lane >> 3, r = min(lane & 7, 5);
  double gs[6], hs[6], a[6];
#pragma unroll
  for (int b = 0; b < 6; b++) {
    gs[b] = st->scale[b] * st->g[b];
    hs[b] = st->scale[r] * st->H[r * 6 + b] * st->scale[b];
  }
  const double hrr = st->scale[r] * st->H[r * 7] * st->scale[r];
  const double dg = st->reuse_diagonal ? st->diag[r] : lm_diag(hrr);
  const double l = sqrt(dg / st->radius);
#pragma unroll
  for (int b = 0; b < 6; b++) {
    const double h = st->H[r * 6 + b];
    a[b] = grp == 1 ? (b == r ? h - eig_thre : h) : (b == r ? hs[b] + l * l : hs[b]);
  }
  double inv[6];
  const bool ok_grp = chol6_rows(a, inv);
  StepTry t;
  t.ok = __shfl_sync(MLOAM_FULL_MASK, (int)ok_grp, 0) != 0;
  t.deg_ok = __shfl_sync(MLOAM_FULL_MASK, (int)ok_grp, 8) != 0 && deg_test;
  t.mcc = 0.0;
#pragma unroll
  for (int j = 0; j < 6; j++) {
    inv[j] = __shfl_sync(MLOAM_FULL_MASK, inv[j], 0);
    t.diag[j] = __shfl_sync(MLOAM_FULL_MASK, dg, j);
    t.step[j] = 0.0;
  }
  if (t.ok) {  // every lane solves with group 0's factor
    double L[36];
#pragma unroll
    for (int i = 1; i < 6; i++)
#pragma unroll
      for (int k = 0; k < i; k++) L[i * 6 + k] = __shfl_sync(MLOAM_FULL_MASK, a[k], i);
    chol6_solve(L, inv, gs, t.step);
#pragma unroll
    for (int j = 0; j < 6; j++) {
      t.step[j] = -t.step[j];
      if (!isfinite(t.step[j])) t.ok = false;
    }
  }
  if (t.ok) {
    double hr = 0;  // row r of Hs times the step
#pragma unroll
    for (int b = 0; b < 6; b++) hr += hs[b] * t.step[b];
    double sg = 0, sHs = 0;
#pragma unroll
    for (int q = 0; q < 6; q++) {
      sg += t.step[q] * gs[q];
      sHs += t.step[q] * __shfl_sync(MLOAM_FULL_MASK, hr, q);
    }
    t.mcc = -(sg + 0.5 * sHs);
    if (t.mcc < 0) t.ok = false;
  }
  return t;
}

// lm_compute_step on the warp.  first / xc_first: the arithmetic of the loop's first pass and its candidate pose, already done by
// the caller (mode 1), or null.
__device__ void lm_compute_step_warp(LMState *st, const StepTry *first, const double *xc_first) {
  const int lane = threadIdx.x & 31;
  while (true) {
    if (st->iteration >= st->max_inner) {
      __syncwarp();
      if (lane == 0) st->done = 1, st->termination = kTermMaxIterations;
      return;
    }
    StepTry t;
    double xc[7];
    if (first) {
      t = *first;
#pragma unroll
      for (int k = 0; k < 7; k++) xc[k] = xc_first[k];
      first = nullptr;
    } else {
      t = lm_try_step_warp(st, false, 0.0);
      if (t.ok) {
        double delta[6];
#pragma unroll
        for (int j = 0; j < 6; j++) delta[j] = t.step[j] * st->scale[j];
        pose_plus(st->x, delta, st->V_update, xc);
      }
    }
    const bool reuse = st->reuse_diagonal != 0;
    const int num_invalid = st->num_invalid + 1;
    const double radius = lm_radius_invalid(st->radius);
    __syncwarp();
    if (lane == 0) {
      if (!reuse)
        for (int j = 0; j < 6; j++) st->diag[j] = t.diag[j];
      st->reuse_diagonal = 1;
      st->iteration++;
      st->total_iterations++;
      if (!t.ok) {
        st->num_invalid = num_invalid;
        if (num_invalid >= kMaxInvalidSteps) st->done = 1, st->termination = kTermInvalidSteps;
        else st->radius = radius;
      } else {
        st->num_invalid = 0;
        for (int k = 0; k < 7; k++) st->xc[k] = xc[k];
        st->model_cost_change = t.mcc;
      }
    }
    __syncwarp();
    if (t.ok || num_invalid >= kMaxInvalidSteps) return;
  }
}

// lm_advance on warp 0 of the tail block (all 32 lanes call it); st is the shared-memory copy of the state.
__device__ void lm_advance_warp(LMState *st, const double *ne, int mode, double eig_thre, int want_eig) {
  const int lane = threadIdx.x & 31;
  const double cost = ne[NE_H + NE_G];
  if (mode == 1) {
    for (int e = lane; e < 36; e += 32) {  // unpack_ne: both triangles take the packed upper entry
      const int i = e / 6, j = e % 6, lo = min(i, j), hi = max(i, j);
      const double h = ne[lo * 6 - lo * (lo - 1) / 2 + hi - lo];
      st->H[e] = h, st->H0[e] = h;
    }
    const int n0 = (int)ne[NE_H + NE_G + 1], n1 = (int)ne[NE_H + NE_G + 2], rows = n0 + n1;
    const bool skip = rows < st->min_corr;
    double x[7];
#pragma unroll
    for (int k = 0; k < 7; k++) x[k] = st->x[k];
    if (lane == 0) {
      for (int i = 0; i < 6; i++) st->g[i] = ne[NE_H + i];
      st->cost = cost, st->initial_cost = cost;
      st->n_valid[0] = n0, st->n_valid[1] = n1, st->rows = rows, st->skipped = 0;
      for (int k = 0; k < 7; k++) st->xc[k] = x[k];
      if (skip) st->done = 1, st->termination = kTermTooFewRows, st->skipped = 1;  // "less correspondence": pose untouched
    }
    if (skip) return;
    bool need_eig = rows > 0 && eig_thre > 0.0;
    const bool deg_test = need_eig && !want_eig;
    double xn = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) xn += x[k] * x[k];
    __syncwarp();  // H
    for (int e = lane; e < 36; e += 32) st->V_update[e] = (e % 7 == 0) ? 1.0 : 0.0;
    if (lane < 6) st->eig[lane] = 0.0, st->scale[lane] = 1.0 / (1.0 + sqrt(st->H[lane * 7]));
    if (lane == 0) {
      st->is_degenerate = 0;
      st->x_norm = sqrt(xn);
      st->radius = kInitialRadius, st->decrease_factor = kDecreaseFactor, st->reuse_diagonal = 0;
      st->iteration = 0, st->num_invalid = 0, st->done = 0, st->termination = kTermMaxIterations;
    }
    __syncwarp();
    // V_update does not enter the step: factor it (group 0) next to the degeneracy test (group 1)
    const StepTry t = lm_try_step_warp(st, deg_test, eig_thre);
    if (t.deg_ok) need_eig = false;
    if (need_eig) {  // (nearly) degenerate, or the eigenvalue report was asked for: the Jacobi solver on one lane
      if (lane == 0) eig_remap(st, eig_thre);
      __syncwarp();
    }
    // gradient_max_norm (even lanes) and the candidate pose of the step (odd lanes), with the final V_update
    double dv[6], xp[7];
#pragma unroll
    for (int j = 0; j < 6; j++) dv[j] = (lane & 1) ? t.step[j] * st->scale[j] : -st->g[j];
    pose_plus(x, dv, st->V_update, xp);
    double m = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) m = fmax(m, fabs(x[k] - xp[k]));
    m = __shfl_sync(MLOAM_FULL_MASK, m, 0);
    double xc[7];
#pragma unroll
    for (int k = 0; k < 7; k++) xc[k] = __shfl_sync(MLOAM_FULL_MASK, xp[k], 1);
    if (m <= kGradTol) {
      if (lane == 0) st->done = 1, st->termination = kTermGradientTol;
      return;
    }
    lm_compute_step_warp(st, &t, xc);
    return;
  }
  // mode 2
  if (st->done) return;
  double x[7], xc[7];
#pragma unroll
  for (int k = 0; k < 7; k++) x[k] = st->x[k], xc[k] = st->xc[k];
  double sn = 0;
#pragma unroll
  for (int k = 0; k < 7; k++) sn += (x[k] - xc[k]) * (x[k] - xc[k]);
  sn = sqrt(sn);
  double rel;
  const int v = lm_verdict(sn, st->x_norm, st->cost, cost, st->model_cost_change, rel);
  if (v >= 0) {
    if (lane == 0) st->done = 1, st->termination = v;
    return;
  }
  if (v == kLMAccept) {
    const double radius = lm_radius_accept(st->radius, rel);
    double xn = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) xn += xc[k] * xc[k];
    double neg[6], xp[7];
#pragma unroll
    for (int j = 0; j < 6; j++) neg[j] = -ne[NE_H + j];
    pose_plus(xc, neg, st->V_update, xp);  // gradient_max_norm at the accepted pose
    double m = 0;
#pragma unroll
    for (int k = 0; k < 7; k++) m = fmax(m, fabs(xc[k] - xp[k]));
    __syncwarp();
    for (int e = lane; e < 36; e += 32) {
      const int i = e / 6, j = e % 6, lo = min(i, j), hi = max(i, j);
      st->H[e] = ne[lo * 6 - lo * (lo - 1) / 2 + hi - lo];
    }
    if (lane == 0) {
      st->radius = radius, st->decrease_factor = kDecreaseFactor, st->reuse_diagonal = 0;
      for (int k = 0; k < 7; k++) st->x[k] = xc[k];
      st->x_norm = sqrt(xn);
      for (int i = 0; i < 6; i++) st->g[i] = ne[NE_H + i];
      st->cost = cost;
      if (m <= kGradTol) st->done = 1, st->termination = kTermGradientTol;
    }
    __syncwarp();
    if (m <= kGradTol) return;
  } else {
    double radius = st->radius, df = st->decrease_factor;
    lm_radius_reject(radius, df);
    __syncwarp();
    if (lane == 0) st->radius = radius, st->decrease_factor = df, st->reuse_diagonal = 1;
    __syncwarp();
  }
  lm_compute_step_warp(st, nullptr, nullptr);
}

// Called by all LM_THREADS threads of one block.  Block partials -> packed normal equations in a fixed order
// (deterministic): warp w sums blocks w, w+8, ... for component `lane`, then the 8 warp sums are added in warp order.
// The LM state lives in global memory between launches; it is staged through shared memory here because the
// state machine touches it a few hundred times (each a dependent L2 round trip otherwise).
//
// Multi-GPU (p2p != nullptr): one LiDAR per GPU, the LM step needs the SUM of every rank's normal equations.  The
// reduction, the exchange and the step are one kernel: this block stores its 30 doubles into slot[rank] of every
// rank's exchange buffer (peer stores over NVLink), raises its flag there, polls its own buffer until all ranks'
// flags carry this exchange's epoch, and adds the slots in rank order — the same order on every rank, so all ranks
// advance bit-identical states.  Slots and flags are double-buffered by the parity of the epoch: a rank can only be
// one exchange ahead of the slowest one, so a slot is never overwritten before it has been read.
//
// SERIAL: the state machine on thread 0 (lm_advance, MLOAM_LM_TAIL=serial) instead of warp 0 (lm_advance_warp); bit-identical.
// Two instances rather than a run-time branch, so that the warp tail does not carry the serial code's registers and stack.
// xc_pub (or null): 7 doubles that receive the new candidate pose, copied from the shared state.

// Words of LMState a tail stages: mode 2 never reads eig or H0 and never writes V_update, eig or H0.
static_assert(sizeof(LMState) % 8 == 0, "LMState is staged as 8-byte words");
constexpr int kStateWords = (int)(sizeof(LMState) / 8);
constexpr int kVupdateWord = (int)(offsetof(LMState, V_update) / 8), kEigWord = (int)(offsetof(LMState, eig) / 8);
constexpr int kH0EndWord = (int)(offsetof(LMState, initial_cost) / 8);
static_assert(kEigWord == kVupdateWord + 36 && kH0EndWord == kEigWord + 6 + 36, "V_update, eig and H0 are adjacent");
__device__ __forceinline__ void stage_state_in(LMState *s, const LMState *gst, int mode, int nthreads) {
  const unsigned long long *src = reinterpret_cast<const unsigned long long *>(gst);
  unsigned long long *dst = reinterpret_cast<unsigned long long *>(s);
  for (int k = threadIdx.x; k < kStateWords; k += nthreads)
    if (mode != 2 || k < kEigWord || k >= kH0EndWord) dst[k] = __ldcg(src + k);
}
__device__ __forceinline__ void stage_state_out(const LMState *s, LMState *gst, int mode, int nthreads) {
  const unsigned long long *src = reinterpret_cast<const unsigned long long *>(s);
  unsigned long long *dst = reinterpret_cast<unsigned long long *>(gst);
  for (int k = threadIdx.x; k < kStateWords; k += nthreads)
    if (mode != 2 || k < kVupdateWord || k >= kH0EndWord) dst[k] = src[k];
}

// Runs the state machine on the staged state s (thread 0 serially, or warp 0) and keeps the cycle counters.  Called by all threads.
template <bool SERIAL>
__device__ __forceinline__ void lm_run(LMState *s, const double *ne, int mode, double eig_thre, int want_eig, long long t0, bool failed) {
  if (threadIdx.x >= 32) return;
  const long long t1 = clock64();
  if (SERIAL) {
    if (threadIdx.x == 0) lm_advance(s, ne, mode, eig_thre, want_eig);
  } else {
    lm_advance_warp(s, ne, mode, eig_thre, want_eig);
    __syncwarp();
  }
  if (threadIdx.x == 0) {
    s->work[0] = 0, s->work[1] = 0;  // re-arm the match work queues
    if (failed) s->done = 1, s->termination = kTermExchangeFailed;  // the peer-memory exchange failed: the state is not trustworthy
    s->dbg_cycles[0] += t1 - t0, s->dbg_cycles[1] += clock64() - t1, s->dbg_cycles[2] += 1;
  }
}

// Shared memory of the tails, at namespace scope so that both instances of a tail in one kernel use the same allocation.
__shared__ double tail_ne[NE_PACK];
__shared__ LMState tail_state;
__shared__ unsigned long long tail_p2p_epoch;
__shared__ int tail_p2p_timeout;
__shared__ double tail_wsum[LM_THREADS / 32][32];

template <bool SERIAL>
__device__ __noinline__ void lm_tail(const double *partials, int n_blocks, LMState *gst, int mode, double eig_thre, int want_eig, double *out_ne,
                                     const P2PView *p2p, double *xc_pub) {
  double *const ne = tail_ne;
  unsigned long long &p2p_epoch = tail_p2p_epoch;
  int &p2p_timeout = tail_p2p_timeout;
  double (*const wsum)[32] = tail_wsum;
  LMState &s = tail_state;
  const long long t0 = clock64();
  if (mode != 0) stage_state_in(&s, gst, mode, LM_THREADS);
  {
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    constexpr int S = LM_THREADS / 32;
    double v = 0.0;
    if (lane < NE_PACK) {
      const double *p = partials + lane;
      int b = w;
      for (; b + 7 * S < n_blocks; b += 8 * S) {  // eight loads in flight, same summation order
        double t[8];
#pragma unroll
        for (int u = 0; u < 8; u++) t[u] = __ldcg(p + (size_t)(b + u * S) * NE_PACK);
#pragma unroll
        for (int u = 0; u < 8; u++) v += t[u];
      }
      for (; b < n_blocks; b += S) v += __ldcg(p + (size_t)b * NE_PACK);
    }
    wsum[w][lane] = v;
    __syncthreads();
    if (threadIdx.x < NE_PACK) {
      double t = 0.0;
#pragma unroll
      for (int ww = 0; ww < S; ww++) t += wsum[ww][threadIdx.x];
      ne[threadIdx.x] = t;
      if (out_ne) out_ne[threadIdx.x] = t;
    }
  }
  __syncthreads();
  if (mode == 0) return;
  if (p2p) {
    const int N = p2p->nranks, me = p2p->rank;
    if (threadIdx.x == 0) p2p_epoch = *p2p->epoch, p2p_timeout = 0;
    __syncthreads();
    const unsigned long long ep = p2p_epoch;
    const int par = (int)(ep & 1ull);
    const unsigned target = (unsigned)(ep + 1ull);
    if (threadIdx.x < NE_PACK)
      for (int q = 0; q < N; q++) reinterpret_cast<volatile double *>(p2p->slots[q])[(par * MLOAM_P2P_MAX_RANKS + me) * 32 + threadIdx.x] = ne[threadIdx.x];
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < N) {
      *reinterpret_cast<volatile unsigned *>(p2p->flags[threadIdx.x] + par * MLOAM_P2P_MAX_RANKS + me) = target;  // notify rank threadIdx.x
      volatile unsigned *mine = reinterpret_cast<volatile unsigned *>(p2p->flags[me] + par * MLOAM_P2P_MAX_RANKS + threadIdx.x);
      const long long w0 = clock64();
      while (true) {
        const unsigned v = *mine;
        if (v == target) break;
        if ((int)(v - target) > 0) {  // the peer is AHEAD of this exchange: the ranks lost lock-step, its slot holds a later sum
          p2p_timeout = 2;
          break;
        }
        if (clock64() - w0 > 6000000000ll) {  // ~3 s: a peer never showed up
          p2p_timeout = 1;
          break;
        }
      }
    }
    __threadfence_system();
    __syncthreads();
    if (threadIdx.x < NE_PACK) {
      double t = 0.0;
      for (int q = 0; q < N; q++) t += reinterpret_cast<volatile double *>(p2p->slots[me])[(par * MLOAM_P2P_MAX_RANKS + q) * 32 + threadIdx.x];
      ne[threadIdx.x] = t;
    }
    if (threadIdx.x == 0) *p2p->epoch = ep + 1ull;
    __syncthreads();
  }
  lm_run<SERIAL>(&s, ne, mode, eig_thre, want_eig, t0, p2p && p2p_timeout);
  __syncthreads();
  stage_state_out(&s, gst, mode, LM_THREADS);
  if (xc_pub && threadIdx.x < 7) xc_pub[threadIdx.x] = s.xc[threadIdx.x];
}

__global__ void __launch_bounds__(LM_THREADS) k_lm(const double *__restrict__ partials, int n_blocks, LMState *st, int mode, double eig_thre,
                                                  int want_eig, double *__restrict__ out_ne, int serial) {
  if (serial) lm_tail<true>(partials, n_blocks, st, mode, eig_thre, want_eig, out_ne, nullptr, nullptr);
  else lm_tail<false>(partials, n_blocks, st, mode, eig_thre, want_eig, out_ne, nullptr, nullptr);
}

// ---------------------------------------------------------------------------------------- candidate evaluation
// k_eval_candidate: pass 1 of k_linearize (evaluation at xc + mode-2 tail) for a solve with max_inner == 1, in blocks small
// enough to run beside the speculative matcher: three k_match_knn CTAs (3 x 256 threads x 72 registers = 55296) leave 10240
// registers of an SM, enough for one block of 64 threads at <= 128 registers (8192).  H at xc is never read with one LM
// iteration (the next Solve's mode 1 overwrites LMState::H, the stats report H0), so only g, cost and the row counts are
// accumulated.  Bit-identical to k_linearize: a thread evaluates the same features (blocks of 64 tile k_linearize's blocks of
// 256), the per-component warp butterfly is the same addition tree as k_linearize's packed one, and the tail adds the warp
// sums in k_linearize's order (8 warps per block, then lm_tail's fixed order over the blocks).
constexpr int CAND_THREADS = 64;
constexpr int NE_CAND = 9;  // g | cost | rows(set 0) | rows(set 1) = NE_PACK components 21..29
constexpr int LIN_WARPS = LIN_THREADS / 32;

__shared__ double cand_bsum[64][NE_CAND];  // per k_linearize block (n_lin_blocks <= 64)
__shared__ double cand_vsum[LM_THREADS / 32][NE_CAND];

template <bool SERIAL>
__device__ __noinline__ void cand_tail(const double *wsums, int n_lin_blocks, LMState *gst, double eig_thre) {
  double (*const bsum)[NE_CAND] = cand_bsum;
  double (*const vsum)[NE_CAND] = cand_vsum;
  double *const ne = tail_ne;
  LMState &s = tail_state;
  const long long t0 = clock64();
  stage_state_in(&s, gst, 2, CAND_THREADS);
  // k_linearize's block partial: its 8 warp sums in warp order
  for (int b = threadIdx.x; b < n_lin_blocks; b += CAND_THREADS) {
#pragma unroll 3
    for (int q = 0; q < NE_CAND; q++) {
      double t[LIN_WARPS];
#pragma unroll
      for (int w = 0; w < LIN_WARPS; w++) t[w] = __ldcg(wsums + (size_t)(b * LIN_WARPS + w) * NE_CAND + q);
      double v = 0.0;
#pragma unroll
      for (int w = 0; w < LIN_WARPS; w++) v += t[w];
      bsum[b][q] = v;
    }
  }
  __syncthreads();
  // lm_tail's order: "warp" w of 8 sums blocks w, w + 8, ...; then the 8 in order (H components: sums of zeros)
  for (int task = threadIdx.x; task < (LM_THREADS / 32) * NE_CAND; task += CAND_THREADS) {
    const int w = task / NE_CAND, q = task % NE_CAND;
    double v = 0.0;
    for (int b = w; b < n_lin_blocks; b += LM_THREADS / 32) v += bsum[b][q];
    vsum[w][q] = v;
  }
  __syncthreads();
  if (threadIdx.x < NE_PACK) {
    double t = 0.0;
    if (threadIdx.x >= NE_H)
#pragma unroll
      for (int w = 0; w < LM_THREADS / 32; w++) t += vsum[w][threadIdx.x - NE_H];
    ne[threadIdx.x] = t;
  }
  __syncthreads();
  lm_run<SERIAL>(&s, ne, 2, eig_thre, 1, t0, false);
  __syncthreads();
  stage_state_out(&s, gst, 2, CAND_THREADS);
}

// grid: LIN_THREADS / CAND_THREADS blocks per k_linearize block; wsums: NE_CAND doubles per warp
__global__ void __launch_bounds__(CAND_THREADS, 8) k_eval_candidate(LinArgs a, double *__restrict__ wsums) {
  __shared__ bool is_last;
  // Programmatic dependent launch: state->done, xc and the valid / coefficient arrays come from k_linearize's pass 0
  cudaGridDependencySynchronize();
  cudaTriggerProgrammaticLaunchCompletion();
  if (a.state->done) return;  // the step of the evaluation at x ended the Solve
  double xs[7];
#pragma unroll
  for (int k = 0; k < 7; k++) xs[k] = a.state->xc[k];
  const PoseR P = make_poser(xs);
  double acc[NE_CAND];
#pragma unroll
  for (int k = 0; k < NE_CAND; k++) acc[k] = 0.0;
  const int G = gridDim.x * blockDim.x, gid = blockIdx.x * blockDim.x + threadIdx.x;
  for (int s = 0; s < a.n_sets; s++) {
    const FeatSetDev fs = a.set[s];
    const int fn = fs.d_n ? min(fs.n, *fs.d_n) : fs.n;
    for (int i = (s & 1) ? G - 1 - gid : gid; i < fn; i += G) {  // k_linearize's assignment
      if (!fs.valid[i] || (fs.mask && !fs.mask[i])) continue;
      double J[6], rho;
      const double r = map_factor_row(P, fs, i, a.sqrt_info, a.huber_a, J, &rho);
#pragma unroll
      for (int k = 0; k < 6; k++) acc[k] += J[k] * r;
      acc[6] += 0.5 * rho;
      if (s == 0) acc[7] += 1.0;
      else acc[8] += 1.0;
    }
  }
#pragma unroll
  for (int k = 0; k < NE_CAND; k++)
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc[k] += __shfl_xor_sync(MLOAM_FULL_MASK, acc[k], o);
  if ((threadIdx.x & 31) == 0) {
    double *w = wsums + (size_t)(gid >> 5) * NE_CAND;
#pragma unroll
    for (int k = 0; k < NE_CAND; k++) w[k] = acc[k];
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) is_last = atomicAdd(a.ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  if (a.lm_serial) cand_tail<true>(wsums, (int)(gridDim.x / (LIN_THREADS / CAND_THREADS)), a.state_rw, a.eig_thre);
  else cand_tail<false>(wsums, (int)(gridDim.x / (LIN_THREADS / CAND_THREADS)), a.state_rw, a.eig_thre);
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) *a.ticket = 0u;
}

__global__ void k_lm_init(LMState *st, const double *pose7, int max_inner, int min_corr, SpecState *spec) {
  cudaGridDependencySynchronize();  // programmatic dependent launch: the kernel before may still read the state and SpecState it resets
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (spec) {  // the first matcher of a solve is blind: any half will do, but sel must be 0 or 1 (fresh memory is not)
      for (int k = 0; k < 7; k++) spec->xc[k] = pose7[k];
      spec->sel = 0;
    }
    for (int k = 0; k < 7; k++) st->x[k] = pose7[k], st->xc[k] = pose7[k];
    st->max_inner = max_inner;
    st->min_corr = min_corr, st->skipped = 0;
    st->done = 0, st->termination = kTermMaxIterations, st->total_iterations = 0, st->iteration = 0;
    st->is_degenerate = 0, st->rows = 0, st->n_valid[0] = st->n_valid[1] = 0;
    st->work[0] = st->work[1] = 0;
    st->cost = 0, st->initial_cost = 0;
    for (int i = 0; i < 36; i++) st->V_update[i] = (i % 7 == 0) ? 1.0 : 0.0, st->H0[i] = 0, st->H[i] = 0;
    for (int i = 0; i < 6; i++) st->eig[i] = 0, st->g[i] = 0;
    for (int i = 0; i < 4; i++) st->dbg_cycles[i] = 0;
  }
}

int lm_init_state(Ctx *c, const double *pose7_host, int max_inner, int min_corr, SpecState *spec, bool pdl) {
  MLOAM_CUDA_OK(c, c->lm_state.reserve(sizeof(LMState) + 64));
  stage_pose(c, pose7_host);
  double *d_stage = c->ctl.as<DevCtl>()->pose;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_stage, c->pinned->pose, 7 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  MLOAM_CUDA_OK(c, launch_chain(pdl, k_lm_init, 1, 32, c->stream, c->lm_state.as<LMState>(), d_stage, max_inner, min_corr, spec));
  c->launches++;
  return MLOAM_OK;
}

// ---------------------------------------------------------------------------------------- pose covariance
// cov_mapping = mat_H.inverse() after the last Solve (lidar_mapper_keyframe.cpp:600-610): LMState::H is the loss-corrected J^T J
// at the accepted x, evaluated with the last association — problem.Evaluate at the pose the Solve returns.  Eigen's 6x6 inverse
// is a partial-pivot LU (first largest |pivot| of the column, rows swapped, multipliers divided by the pivot, rank-1 update of the
// trailing block) followed by L U X = P I solved column by column.  A last evaluation with no residual rows gives zeros (Eigen
// would return inf / NaN there).  The speculative schedule keeps the two-pass k_linearize for the last GN iteration, so H is
// accumulated at the final candidate too (k_eval_candidate does not accumulate H).
__global__ void k_pose_cov(const LMState *__restrict__ st, double *__restrict__ out) {
  cudaGridDependencySynchronize();  // programmatic dependent launch: H and rows come from the last k_linearize's tail
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (st->rows <= 0) {
    for (int i = 0; i < 36; i++) out[i] = 0.0;
    return;
  }
  double A[36];
  int perm[6];
  for (int i = 0; i < 36; i++) A[i] = st->H[i];
  for (int i = 0; i < 6; i++) perm[i] = i;
  for (int k = 0; k < 6; k++) {
    int piv = k;
    double best = fabs(A[k * 6 + k]);
    for (int i = k + 1; i < 6; i++)
      if (fabs(A[i * 6 + k]) > best) best = fabs(A[i * 6 + k]), piv = i;
    if (piv != k) {
      for (int j = 0; j < 6; j++) {
        const double t = A[k * 6 + j];
        A[k * 6 + j] = A[piv * 6 + j], A[piv * 6 + j] = t;
      }
      const int t = perm[k];
      perm[k] = perm[piv], perm[piv] = t;
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

int pose_cov_device(Ctx *c, bool pdl) {
  MLOAM_CUDA_OK(c, c->pose_cov.reserve(36 * sizeof(double)));
  MLOAM_CUDA_OK(c, launch_chain(pdl, k_pose_cov, 1, 32, c->stream, c->lm_state.as<const LMState>(), c->pose_cov.as<double>()));
  c->launches++;
  return MLOAM_OK;
}

// What k_linearize and k_eval_candidate share: the feature sets, the grid (k_eval_candidate runs LIN_THREADS / CAND_THREADS
// blocks per k_linearize block) and c->partials = [NE_PACK doubles per k_linearize block, max_nb + 2 of them][ticket +
// generation word][NE_CAND doubles per k_eval_candidate warp].
static int lin_setup(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, double eig_thre, LinArgs &a, int *nb_out,
                     double **wsums) {
  memset(&a, 0, sizeof(a));
  int n_total = 0;
  for (int s = 0; s < 2; s++) {
    if (s < n_sets) {
      a.set[s].pts = sets[s].pts, a.set[s].valid = sets[s].valid, a.set[s].coeff = sets[s].coeff;
      a.set[s].n = sets[s].n, a.set[s].is_plane = sets[s].is_plane, a.set[s].d_n = sets[s].d_n;
      a.set[s].sinfo = sets[s].sinfo, a.set[s].mask = sets[s].mask;
      n_total = sets[s].n > n_total ? sets[s].n : n_total;
    } else {
      a.set[s].pts = nullptr, a.set[s].valid = nullptr, a.set[s].coeff = nullptr, a.set[s].n = 0, a.set[s].is_plane = 0, a.set[s].d_n = nullptr;
      a.set[s].sinfo = nullptr, a.set[s].mask = nullptr;
    }
  }
  a.n_sets = n_sets, a.sqrt_info = sqrt_info, a.huber_a = huber_a;
  a.state = c->lm_state.as<LMState>();
  a.state_rw = c->lm_state.as<LMState>();
  a.eig_thre = eig_thre;
  a.lm_serial = c->lm_tail_serial;
  int nb = (n_total + LIN_THREADS - 1) / LIN_THREADS;
  if (nb < 1) nb = 1;
  // n_total is a launch upper bound (device-side counts are usually far smaller): 64 blocks x 256 threads cover a
  // typical frame's ~10^4 features one per thread, and the tail's fixed-order sum reads 64 partials in one round.
  const int max_nb = c->sm_count;
  if (nb > max_nb) nb = max_nb;
  if (nb > 64) nb = 64;
  const size_t wsums_at = (size_t)NE_PACK * (max_nb + 3);
  MLOAM_CUDA_OK(c, c->partials.reserve(sizeof(double) * (wsums_at + (size_t)NE_CAND * 64 * LIN_WARPS)));
  a.ticket = reinterpret_cast<unsigned *>(c->partials.as<double>() + (size_t)NE_PACK * (max_nb + 2));
  if (c->ticket_zeroed_for != c->partials.p) {  // a fresh partials buffer: the last-block ticket starts at zero
    MLOAM_CUDA_OK(c, cudaMemsetAsync(a.ticket, 0, sizeof(double), c->stream));
    c->ticket_zeroed_for = c->partials.p;
  }
  *nb_out = nb;
  *wsums = c->partials.as<double>() + wsums_at;
  return MLOAM_OK;
}

int linearize_device(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, const double *d_pose7,
                     int use_state, int lm_mode, double *d_out30, const LinOpts &o, bool *two_pass_done) {
  LinArgs a;
  int nb = 0;
  double *wsums = nullptr;
  int rc = lin_setup(c, sets, n_sets, sqrt_info, huber_a, o.eig_thre, a, &nb, &wsums);
  if (rc) return rc;
  const int max_nb = c->sm_count;
  a.pose = d_pose7;
  a.use_state = use_state;
  a.respect_done = (lm_mode == 2) ? 1 : 0;
  const bool collective = c->nccl_comm && o.collective;  // sum over the ranks wanted for this solve
  const bool fused = lm_mode != 0 && (!collective || c->p2p_on) && !d_out30;
  // only the collective solves (scan2map on every rank in lock-step) exchange; per-rank solves on the same context — the tracker,
  // mloam_normal_equations — stay local
  a.p2p = (fused && c->p2p_on && o.collective) ? static_cast<const P2PView *>(c->p2p_view) : nullptr;
  a.lm_mode = fused ? lm_mode : 0, a.want_eig = o.want_eig;
  // both evaluations of an LM iteration in one launch: only with the fused tail (the barrier is released by the block that ran it)
  a.two_pass = (o.two_pass && fused && lm_mode == 1) ? 1 : 0;
  if (two_pass_done) *two_pass_done = a.two_pass != 0;
  // the speculative schedule's commit rides in the fused tail of the evaluation at x
  if (o.spec && !(fused && lm_mode == 1 && !a.p2p)) {
    c->err = "linearize: the speculative schedule needs the fused single-GPU evaluation at x";
    return MLOAM_E_STATE;
  }
  a.spec = o.spec, a.spec_publish = o.spec_publish ? 1 : 0;
  // a fit the matcher deferred to this evaluation
  int kfit = 0;
  if (o.fit && o.fit->K) {
    if (lm_mode != 1 || n_sets != 2 || (o.fit->K != 5 && o.fit->K != 10)) {
      c->err = "linearize: a deferred fit is pending but this is not the first evaluation of a solve";
      return MLOAM_E_STATE;
    }
    kfit = o.fit->K;
    a.fit[0] = o.fit->set[0], a.fit[1] = o.fit->set[1];
    a.fit_min_plane_dis = o.fit->min_plane_dis, a.fit_check_fov = o.fit->check_fov;
  }
  // phase stamps of the evaluations at x of a fused solve, one slot each (scan2map_enqueue restarts the count)
  if (c->lin_trace_on && fused && lm_mode == 1 && c->lin_trace_n < LIN_TRACE_SLOTS) {
    const size_t bytes = sizeof(unsigned long long) * LIN_TRACE_SLOT * LIN_TRACE_SLOTS;
    if (c->lin_trace.cap < bytes) {
      MLOAM_CUDA_OK(c, c->lin_trace.reserve(bytes));
      MLOAM_CUDA_OK(c, cudaMemsetAsync(c->lin_trace.p, 0, c->lin_trace.cap, c->stream));
    }
    a.trace = c->lin_trace.as<unsigned long long>() + (size_t)LIN_TRACE_SLOT * c->lin_trace_n++;
  }
  {
    ProfScope ps(c, "linearize");
    double *const pt = c->partials.as<double>();
    void (*k)(LinArgs, double *);
    if (a.trace) k = kfit == 5 ? k_linearize<5, true> : (kfit == 10 ? k_linearize<10, true> : k_linearize<0, true>);
    else k = kfit == 5 ? k_linearize<5> : (kfit == 10 ? k_linearize<10> : k_linearize<0>);
    MLOAM_CUDA_OK(c, launch_chain(o.pdl, k, nb, LIN_THREADS, c->stream, a, pt));
    c->launches++;
  }
  if (fused) {
    MLOAM_CUDA_OK(c, cudaGetLastError());
    return MLOAM_OK;
  }
  if (collective && lm_mode != 0) {
    // multi-GPU: rank-local sum -> NCCL all-reduce of the 30 packed doubles -> identical LM step on every rank
    double *ne = c->partials.as<double>() + (size_t)NE_PACK * max_nb;
    {
      ProfScope ps(c, "lm");
      k_lm<<<1, LM_THREADS, 0, c->stream>>>(c->partials.as<double>(), nb, c->lm_state.as<LMState>(), 0, 0.0, 0, ne, c->lm_tail_serial);
      c->launches++;
    }
    int rc = comm_allreduce_doubles(c, ne, NE_PACK);
    if (rc) return rc;
    ProfScope ps(c, "lm");
    k_lm<<<1, LM_THREADS, 0, c->stream>>>(ne, 1, c->lm_state.as<LMState>(), lm_mode, o.eig_thre, o.want_eig, d_out30, c->lm_tail_serial);
    c->launches++;
  } else {
    ProfScope ps(c, "lm");
    k_lm<<<1, LM_THREADS, 0, c->stream>>>(c->partials.as<double>(), nb, c->lm_state.as<LMState>(), lm_mode, o.eig_thre, o.want_eig, d_out30, c->lm_tail_serial);
    c->launches++;
  }
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

int eval_candidate_device(Ctx *c, const FeatSet *sets, int n_sets, double sqrt_info, double huber_a, double eig_thre, bool pdl) {
  LinArgs a;
  int nb = 0;
  double *wsums = nullptr;
  int rc = lin_setup(c, sets, n_sets, sqrt_info, huber_a, eig_thre, a, &nb, &wsums);
  if (rc) return rc;
  ProfScope ps(c, "candidate");
  MLOAM_CUDA_OK(c, launch_chain(pdl, k_eval_candidate, nb * (LIN_THREADS / CAND_THREADS), CAND_THREADS, c->stream, a, wsums));
  c->launches++;
  return MLOAM_OK;
}

// ---------------------------------------------------------------------------------------- batched Evaluate
__global__ void k_factor_evaluate(int kind, int n, const double *__restrict__ points, const double *__restrict__ coeffs,
                                  const double *__restrict__ sqrt_info, const double *__restrict__ params,
                                  double *__restrict__ res, double *__restrict__ jac) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const D3 p{points[i * 3], points[i * 3 + 1], points[i * 3 + 2]};
  const double *cf = coeffs + (size_t)i * 6;
  const double s = sqrt_info ? sqrt_info[i] : 1.0;
  const D3 c0{cf[0], cf[1], cf[2]}, c1{cf[3], cf[4], cf[5]};
  if (kind <= 1) {
    const PoseR P = make_poser(params);
    double J[6];
    const double r = kind == 0 ? plane_factor(P, p, c0, cf[3], s, J, jac != nullptr) : edge_factor(P, p, c0, c1, s, J, jac != nullptr);
    res[i] = r;
    if (jac) {
      for (int k = 0; k < 6; k++) jac[(size_t)i * 7 + k] = J[k];
      jac[(size_t)i * 7 + 6] = 0.0;
    }
  } else if (kind == 2) {
    const PoseR P = make_poser(params);
    double r[3], J[18];
    edge_vector_factor(P, p, c0, c1, r, J, jac != nullptr);
    for (int k = 0; k < 3; k++) res[(size_t)i * 3 + k] = r[k];
    if (jac)
      for (int a = 0; a < 3; a++) {
        for (int k = 0; k < 6; k++) jac[(size_t)i * 21 + a * 7 + k] = J[a * 6 + k];
        jac[(size_t)i * 21 + a * 7 + 6] = 0.0;
      }
  } else {
    const Chain c = make_chain(params, params + 7, params + 14);
    double Jp[6], Ji[6], Je[6];
    const bool wj = jac != nullptr;
    const double r = kind == 3 ? odom_plane_factor(c, p, c0, cf[3], s, wj ? Jp : nullptr, wj ? Ji : nullptr, wj ? Je : nullptr)
                               : odom_edge_factor(c, p, c0, c1, s, wj ? Jp : nullptr, wj ? Ji : nullptr, wj ? Je : nullptr);
    res[i] = r;
    if (jac) {
      double *o = jac + (size_t)i * 21;
      for (int k = 0; k < 6; k++) o[k] = Jp[k], o[7 + k] = Ji[k], o[14 + k] = Je[k];
      o[6] = o[13] = o[20] = 0.0;
    }
  }
}

int factor_evaluate_device(Ctx *c, int kind, int n, const double *d_points, const double *d_coeffs, const double *d_sqrt_info,
                           const double *d_params, double *d_res, double *d_jac) {
  if (kind < 0 || kind > 4) {
    c->err = "factor_evaluate: kind must be 0..4";
    return MLOAM_E_INVALID;
  }
  if (n <= 0) return MLOAM_OK;
  k_factor_evaluate<<<(n + 127) / 128, 128, 0, c->stream>>>(kind, n, d_points, d_coeffs, d_sqrt_info, d_params, d_res, d_jac);
  c->launches++;
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

}  // namespace mloam
