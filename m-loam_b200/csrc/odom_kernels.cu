// odom_kernels.cu — the odometry node's local-map residuals (Estimator::optimizeMap, estimator.cpp:687-848):
// LidarPureOdom{PlaneNorm,Edge}Factor on the pose chain (pose_pivot [constant], pose_i, ext_n), Huber(1.0),
// ceres::Solve(DENSE_SCHUR, NUM_ITERATIONS).  Each feature emits one row over the FREE blocks:
//   1x6  (pose_i free, ext constant: ESTIMATE_EXTRINSIC == 0, estimator.cpp:640,794-848)
//   1x6  (ext free only)
//   1x12 [J_pose_i | J_ext]  (both free)
// k_odom_linearize<D>: one thread per feature computes (r, row); the D(D+1)/2 + D + 2 packed sums are reduced
// element by element with warp shuffles into a per-warp shared-memory accumulator (a 1x12 row would need 92 fp64
// accumulators per thread otherwise), summed across warps in fixed order, one partial per CTA — no atomics.
// k_odom_lm<D>: fixed-order partial sum + lm.cuh's Levenberg-Marquardt state machine on the odometry problem, D = 6 or 12
// (two 6-dof blocks, PoseLocalParameterization::Plus per block).
#include "ctx.h"
#include "factors.cuh"
#include "host_util.h"
#include "lm.cuh"

namespace mloam {

constexpr int OD_THREADS = 256;

template <int D>
struct OdPack {
  static constexpr int NH = D * (D + 1) / 2;
  static constexpr int N = NH + D + 2;  // H upper | g | cost | rows
};

struct OdomState {
  double xp[7];                // pivot (constant)
  double x[14], xc[14];        // [pose_i | ext]: accepted, candidate
  double H[144], g[12], cost;
  double scale[12], diag[12];
  double radius, decrease_factor, model_cost_change, x_norm, initial_cost;
  int free_mask;               // bit 0: pose_i free, bit 1: ext free
  int reuse_diagonal, iteration, num_invalid, done, termination, total_iterations, rows, max_inner, pad;
};

// Rows: LidarPureOdom* on (pivot, pose_i, ext) with the free blocks of OdomState::free_mask; set 0 corner, 1 surf.
constexpr int OD_SETS = 2;
struct OdomSets {
  const float4 *pts[OD_SETS];
  const float *coeff[OD_SETS];
  int n[OD_SETS];
  int is_plane[OD_SETS];
  double sqrt_info, huber_a;
};

template <int D>
__global__ void __launch_bounds__(OD_THREADS) k_odom_linearize(OdomSets a, const OdomState *st, int use_candidate, double *__restrict__ partials) {
  constexpr int N = OdPack<D>::N, NH = OdPack<D>::NH;
  __shared__ double acc[OD_THREADS / 32][N];
  if (use_candidate && st->done) return;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  for (int k = lane; k < N; k += 32) acc[wid][k] = 0.0;
  __syncwarp();
  const Chain ch = make_chain(st->xp, use_candidate ? st->xc : st->x, use_candidate ? st->xc + 7 : st->x + 7);
  const int fm = st->free_mask;
  for (int s = 0; s < OD_SETS; s++) {
    const int n = a.n[s];
    if (n <= 0) continue;
    // all lanes of a warp iterate together (the shuffles below need them); out-of-range lanes contribute zeros
    for (int base = (blockIdx.x * (OD_THREADS / 32) + wid) * 32; base < n; base += gridDim.x * OD_THREADS) {
      const int i = base + lane;
      double row[D];
#pragma unroll
      for (int k = 0; k < D; k++) row[k] = 0.0;
      double r = 0.0, rho = 0.0, one = 0.0;
      if (i < n) {
        const float4 pf = __ldg(a.pts[s] + i);
        const D3 p{(double)pf.x, (double)pf.y, (double)pf.z};
        const float *cf = a.coeff[s] + (size_t)i * 6;
        double Ji[6], Je[6];
        const D3 c0{(double)cf[0], (double)cf[1], (double)cf[2]}, c1{(double)cf[3], (double)cf[4], (double)cf[5]};
        if (a.is_plane[s]) r = odom_plane_factor(ch, p, c0, (double)cf[3], a.sqrt_info, nullptr, Ji, Je);
        else r = odom_edge_factor(ch, p, c0, c1, a.sqrt_info, nullptr, Ji, Je);
        double rho1;
        huber(a.huber_a, r * r, &rho, &rho1);
        const double sc = sqrt(rho1);
        r = sc * r;
        if (D == 12) {
#pragma unroll
          for (int k = 0; k < 6; k++) row[k] = sc * Ji[k], row[6 + k] = sc * Je[k];
        } else {
#pragma unroll
          for (int k = 0; k < 6; k++) row[k] = sc * ((fm & 1) ? Ji[k] : Je[k]);
        }
        one = 1.0;
      }
      // element-wise warp reduction into the warp's accumulator (lane 0 adds; order fixed => deterministic)
      int q = 0;
#pragma unroll
      for (int i0 = 0; i0 < D; i0++) {
#pragma unroll
        for (int j0 = i0; j0 < D; j0++) {
          double v = row[i0] * row[j0];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(MLOAM_FULL_MASK, v, o);
          if (lane == 0) acc[wid][q] += v;
          q++;
        }
      }
#pragma unroll
      for (int k = 0; k < D + 2; k++) {
        double v = k < D ? row[k] * r : (k == D ? 0.5 * rho : one);
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(MLOAM_FULL_MASK, v, o);
        if (lane == 0) acc[wid][NH + k] += v;
      }
    }
  }
  __syncthreads();
  for (int k = threadIdx.x; k < N; k += OD_THREADS) {
    double v = 0.0;
#pragma unroll
    for (int w = 0; w < OD_THREADS / 32; w++) v += acc[w][k];
    partials[(size_t)blockIdx.x * N + k] = v;
  }
}

// ------------------------------------------------------------------------------------------ LM (D = 6 | 12)
// The odometry problem of the single-thread machine (lm.cuh): x (+) delta over the free blocks with the identity V_update (the
// odometry's per-block degeneracy remap, estimator.cpp:1610-1635, is not applied here — next tier), chol<D>.
template <int D_>
struct OdomProblem {
  using State = OdomState;
  static constexpr int D = D_, NX = 14;
  __device__ static bool solve(double *A, const double *b, double *x) {
    if (!chol<D>(A)) return false;
    chol_solve<D>(A, b, x);
    return true;
  }
  __device__ static void plus_into(const OdomState *st, const double *delta, double *out) {
    const double I6[36] = {1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1, 0, 0, 0, 0, 0, 0, 1};
    for (int k = 0; k < 14; k++) out[k] = st->x[k];
    if (D == 12) {
      pose_plus(st->x, delta, I6, out);
      pose_plus(st->x + 7, delta + 6, I6, out + 7);
    } else if (st->free_mask & 1) {
      pose_plus(st->x, delta, I6, out);
    } else {
      pose_plus(st->x + 7, delta, I6, out + 7);
    }
  }
  __device__ static void plus(OdomState *st, const double *delta) { plus_into(st, delta, st->xc); }
  __device__ static double x_norm(const OdomState *st) {  // the free blocks, pose_i then ext
    double s = 0;
    if (D == 12 || (st->free_mask & 1))
      for (int k = 0; k < 7; k++) s += st->x[k] * st->x[k];
    if (D == 12 || (st->free_mask & 2))
      for (int k = 7; k < 14; k++) s += st->x[k] * st->x[k];
    return sqrt(s);
  }
  __device__ static double grad_max(const OdomState *st) {
    double neg[D], xo[14];
    for (int j = 0; j < D; j++) neg[j] = -st->g[j];
    plus_into(st, neg, xo);
    double m = 0;
    for (int k = 0; k < 14; k++) m = fmax(m, fabs(st->x[k] - xo[k]));
    return m;
  }
};

template <int D>
__global__ void __launch_bounds__(OD_THREADS) k_odom_lm(const double *__restrict__ partials, int n_blocks, OdomState *st, int mode) {
  constexpr int N = OdPack<D>::N, NH = OdPack<D>::NH;
  __shared__ double ne[N];
  for (int k = threadIdx.x; k < N; k += OD_THREADS) {
    double v = 0.0;
    for (int b = 0; b < n_blocks; b++) v += partials[(size_t)b * N + k];
    ne[k] = v;
  }
  __syncthreads();
  if (threadIdx.x != 0) return;
  double H[D * D], g[D];
  int q = 0;
  for (int i = 0; i < D; i++)
    for (int j = i; j < D; j++) H[i * D + j] = H[j * D + i] = ne[q++];
  for (int k = 0; k < D; k++) g[k] = ne[NH + k];
  const double cost = ne[NH + D];
  if (mode == 2) {
    lm_digest<OdomProblem<D>>(st, H, g, cost);
    return;
  }
  for (int i = 0; i < D * D; i++) st->H[i] = H[i];
  for (int i = 0; i < D; i++) st->g[i] = g[i];
  st->cost = st->initial_cost = cost;
  st->rows = (int)ne[NH + D + 1];
  lm_begin<OdomProblem<D>>(st);
}

__global__ void k_odom_init(OdomState *st, const double *x21, int free_mask, int max_inner) {
  if (threadIdx.x == 0) {
    for (int k = 0; k < 7; k++) st->xp[k] = x21[k];
    for (int k = 0; k < 14; k++) st->x[k] = st->xc[k] = x21[7 + k];
    st->free_mask = free_mask, st->max_inner = max_inner;
    st->done = 0, st->termination = kTermMaxIterations, st->total_iterations = 0, st->iteration = 0, st->rows = 0, st->cost = st->initial_cost = 0;
  }
}

template <int D>
static int odom_solve_run(Ctx *c, const OdomSets &sets, OdomState *st, int max_inner, int nb, double *partials) {
  int *h_done = &c->pinned->done;
  k_odom_linearize<D><<<nb, OD_THREADS, 0, c->stream>>>(sets, st, 0, partials);
  k_odom_lm<D><<<1, OD_THREADS, 0, c->stream>>>(partials, nb, st, 1);
  c->launches += 2;
  for (int it = 0; it < max_inner; it++) {
    k_odom_linearize<D><<<nb, OD_THREADS, 0, c->stream>>>(sets, st, 1, partials);
    k_odom_lm<D><<<1, OD_THREADS, 0, c->stream>>>(partials, nb, st, 2);
    c->launches += 2;
    MLOAM_CUDA_OK(c, cudaMemcpyAsync(h_done, &st->done, sizeof(int), cudaMemcpyDeviceToHost, c->stream));
    MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
    if (*h_done) break;
  }
  MLOAM_CUDA_OK(c, cudaGetLastError());
  return MLOAM_OK;
}

static_assert(sizeof(OdomState) <= sizeof(PinnedBlock::odom), "OdomState mirror in the pinned block");
static OdomState *odom_mirror(Ctx *c) { return reinterpret_cast<OdomState *>(c->pinned->odom); }

// Ctx::odom_work: OdomState, then the packed equations of nb blocks
static int odom_work(Ctx *c, int nb, OdomState **st, double **partials) {
  MLOAM_CUDA_OK(c, carve(c->odom_work, [&](Carve &cv) {
    *st = cv.take<OdomState>(1);
    *partials = cv.take<double>(OdPack<12>::N * (size_t)nb);
  }));
  return MLOAM_OK;
}

}  // namespace mloam

using namespace mloam;

extern "C" int mloam_odom_solve(mloam_ctx_t *h, int n, const unsigned char *h_types, const double *h_points, const double *h_coeffs,
                                const double *pose_pivot7, double *pose_i7, double *ext7, int free_mask, int max_iterations,
                                double huber_a, double sqrt_info, mloam_solve_stats_t *stats) {
  if (!h || n < 0 || !pose_pivot7 || !pose_i7 || !ext7 || free_mask < 1 || free_mask > 3 || (n > 0 && (!h_types || !h_points || !h_coeffs)))
    return MLOAM_E_INVALID;
  Ctx *c = &h->c;
  cudaSetDevice(c->device);
  if (stats) memset(stats, 0, sizeof(*stats));
  // PointPlaneFeature carries float-valued point_/coeffs_ (feature_extract.hpp:771-781,872-875): device feature format
  std::vector<float4> pts[2];
  std::vector<float> cf[2];
  for (int i = 0; i < n; i++) {
    const int t = h_types[i] == 's' ? 1 : 0;
    pts[t].push_back(make_float4((float)h_points[i * 3], (float)h_points[i * 3 + 1], (float)h_points[i * 3 + 2], 0.f));
    for (int k = 0; k < 6; k++) cf[t].push_back((float)h_coeffs[(size_t)i * 6 + k]);
  }
  OdomSets sets;
  memset(&sets, 0, sizeof(sets));
  int n_max = 0;
  for (int t = 0; t < 2; t++) {
    const int nt = (int)pts[t].size();
    MLOAM_CUDA_OK(c, c->scan_pts[t].reserve(sizeof(float4) * (size_t)(nt + 1)));
    int rc = reserve_feat(c, t, nt);
    if (rc) return rc;
    if (nt > 0) {
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->scan_pts[t].p, pts[t].data(), sizeof(float4) * nt, cudaMemcpyHostToDevice, c->stream));
      MLOAM_CUDA_OK(c, cudaMemcpyAsync(c->feat_coeff[t].p, cf[t].data(), sizeof(float) * 6 * nt, cudaMemcpyHostToDevice, c->stream));
    }
    sets.pts[t] = c->scan_pts[t].as<float4>(), sets.coeff[t] = c->feat_coeff[t].as<float>(), sets.n[t] = nt, sets.is_plane[t] = t;
    n_max = nt > n_max ? nt : n_max;
  }
  sets.sqrt_info = sqrt_info, sets.huber_a = huber_a;
  const int D = free_mask == 3 ? 12 : 6;
  int nb = (n_max + OD_THREADS - 1) / OD_THREADS;
  nb = nb < 1 ? 1 : (nb > c->sm_count ? c->sm_count : nb);
  OdomState *st;
  double *partials;
  int rc = odom_work(c, nb, &st, &partials);
  if (rc) return rc;
  double *stage = c->pinned->odom_x;
  for (int k = 0; k < 7; k++) stage[k] = pose_pivot7[k], stage[7 + k] = pose_i7[k], stage[14 + k] = ext7[k];
  double *d_x = c->ctl.as<DevCtl>()->odom_x;
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(d_x, stage, 21 * sizeof(double), cudaMemcpyHostToDevice, c->stream));
  k_odom_init<<<1, 32, 0, c->stream>>>(st, d_x, free_mask, max_iterations);
  c->launches++;
  rc = D == 12 ? odom_solve_run<12>(c, sets, st, max_iterations, nb, partials) : odom_solve_run<6>(c, sets, st, max_iterations, nb, partials);
  if (rc) return rc;
  OdomState *hs = odom_mirror(c);
  MLOAM_CUDA_OK(c, cudaMemcpyAsync(hs, st, sizeof(OdomState), cudaMemcpyDeviceToHost, c->stream));
  MLOAM_CUDA_OK(c, cudaStreamSynchronize(c->stream));
  for (int k = 0; k < 7; k++) pose_i7[k] = hs->x[k], ext7[k] = hs->x[7 + k];
  if (stats) {
    stats->ran = 1, stats->lm_iterations = hs->total_iterations, stats->termination = hs->termination;
    stats->final_cost = hs->cost, stats->n_surf = (int)pts[1].size(), stats->n_corner = (int)pts[0].size();
    for (int i = 0; i < 6; i++)
      for (int j = 0; j < 6; j++) stats->H[i * 6 + j] = hs->H[i * D + j];  // leading 6x6 block
  }
  return MLOAM_OK;
}
